"""SDXL text-slider trainer — same command line as the reference's trainscripts/textsliders/train_lora_xl.py:418-474:

    python trainscripts/textsliders/train_lora_xl.py --attributes 'male, female' --name 'agesliderXL' --rank 4 \
        --alpha 1 --config_file 'trainscripts/textsliders/data/config-xl.yaml'
    torchrun --nproc-per-node 4 trainscripts/textsliders/train_lora_xl.py ...     # one conditioned prediction per GPU

The loop runs in sliders_b200 (sm_90a kernels; needs an H100).  See sliders_b200/cli.py for the offline flags."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from sliders_b200 import cli  # noqa: E402

if __name__ == "__main__":
    cli.main("text_xl")
