"""Generates the clip-length fixtures tests/golden/ref_{tiny12,tiny5,c2mini24}.npz by running the UNMODIFIED reference on
the CPU, through oracle/gen_golden.py's writer (same inputs, same checks: regenerating must reproduce every committed
tensor bit for bit). TEST INFRASTRUCTURE: needs the reference tree, like oracle/gen_golden.py.

  python scripts/gen_golden_video_length.py [tiny12 tiny5 c2mini24]

The cases are clip lengths off the 8 / 16 / 32-frame tiles of the temporal-attention kernels (t2v_video_sample.py --L):
12 frames run ragged in a 16-frame tile, 5 frames (odd) in an 8-frame tile, 24 frames at SD1.5 widths in a 32-frame
tile (two 16-row query tiles).
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import gen_golden  # noqa: E402
from oracle.gen_golden import BASE  # noqa: E402

CASES = {
    # name: (unet config name, inference cfg, input seed), as oracle/gen_golden.py's CASES
    "tiny12": ("tiny", dict(BASE, inference_steps=5, guidance_steps=3, guidance_scale=0.4, video_length=12, height=128,
                            width=128, warm_up_steps=2, cool_up_steps=2), 92),
    "tiny5": ("tiny", dict(BASE, inference_steps=4, guidance_steps=2, guidance_scale=0.3, video_length=5, height=128,
                           width=128), 102),
    "c2mini24": ("sd15", dict(BASE, inference_steps=4, guidance_steps=2, guidance_scale=0.4, video_length=24, height=128,
                              width=128, warm_up_steps=2, cool_up_steps=2), 112),
}

if __name__ == "__main__":
    names = sys.argv[1:] or list(CASES)
    unknown = [n for n in names if n not in CASES]
    if unknown:
        raise SystemExit(f"unknown case(s) {unknown}; choose from {list(CASES)}")
    gen_golden.CASES.update(CASES)
    gen_golden.main(names)
