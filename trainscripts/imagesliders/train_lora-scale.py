"""SD1.x image-slider trainer — same command line as the reference's trainscripts/imagesliders/train_lora-scale.py:

    python trainscripts/imagesliders/train_lora-scale.py --name 'eyeslider' --rank 4 --alpha 1 \
        --config_file 'trainscripts/imagesliders/data/config.yaml' --folder_main 'datasets/eyesize/' \
        --folders 'bigsize, smallsize' --scales '1, -1'

`folder_main/<folder>/` holds images (encoded each iteration by the VAE of `--vae`, default the model directory's) or
VAE-encoded latents (`<name>.pt`), see sliders_b200/cli.py.  Needs an H100."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from sliders_b200 import cli  # noqa: E402

if __name__ == "__main__":
    cli.main("image")
