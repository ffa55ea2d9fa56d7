"""SDXL slider scale sweep over a prompts CSV — same command line as the reference's eval-scripts/generate_images_xl.py:

    python eval-scripts/generate_images_xl.py --model_name 'models/ageslider_alpha1.0_rank4_noxattn/..._last.pt' \
        --prompts_path prompts/prompts-person.csv --save_path out/ --embeds person_embeds.pt

The denoise loop runs in sliders_b200 (sm_90a kernels; needs an H100).  See sliders_b200/eval_sweep.py."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sliders_b200 import eval_sweep  # noqa: E402

if __name__ == "__main__":
    eval_sweep.main(xl=True)
