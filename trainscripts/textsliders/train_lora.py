"""SD1.x text-slider trainer — same command line as the reference's trainscripts/textsliders/train_lora.py:376-429:

    python trainscripts/textsliders/train_lora.py --attributes 'male, female' --name 'ageslider' --rank 4 --alpha 1 \
        --config_file 'trainscripts/textsliders/data/config.yaml'

The loop runs in sliders_b200 (sm_90a kernels; needs an H100).  See sliders_b200/cli.py for the offline flags."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from sliders_b200 import cli  # noqa: E402

if __name__ == "__main__":
    cli.main("text")
