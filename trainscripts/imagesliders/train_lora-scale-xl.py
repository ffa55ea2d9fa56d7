"""SDXL image-slider trainer — same command line as the reference's trainscripts/imagesliders/train_lora-scale-xl.py:465-543:

    python trainscripts/imagesliders/train_lora-scale-xl.py --name 'eyesliderXL' --rank 4 --alpha 1 \
        --config_file 'trainscripts/imagesliders/data/config-xl.yaml' --folder_main 'datasets/eyesize/' \
        --folders 'bigsize, smallsize' --scales '1, -1'

`folder_main/<folder>/` holds VAE-encoded latents (`<name>.pt`), see sliders_b200/cli.py.  Needs an H100."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from sliders_b200 import cli  # noqa: E402

if __name__ == "__main__":
    cli.main("image_xl")
