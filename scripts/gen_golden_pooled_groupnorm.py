"""Generates the frame-pooled GroupNorm fixtures tests/golden/ref_{tiny8,tiny12,c2mini}_pooledgn.npz by running the
UNMODIFIED reference on the CPU with use_inflated_groupnorm=False, through oracle/gen_golden.py's writer (same inputs,
same checks: regenerating must reproduce every committed tensor bit for bit). TEST INFRASTRUCTURE: needs the reference
tree, like oracle/gen_golden.py.

  python scripts/gen_golden_pooled_groupnorm.py [tiny8_pooledgn tiny12_pooledgn c2mini_pooledgn]

In that mode the reference's resnet norms and output norm are torch.nn.GroupNorm on the 5-D [b, c, f, h, w] tensor
(models/resnet.py:143-146, 162-165, models/unet.py:244-247): statistics pooled over the f frames of a batch element.
The writer picks the UNet config by the names "tiny" / "sd15"; while these cases run, those names point at the pooled
configs (same state-dict keys and shapes), and the config name is recorded in each fixture's meta as "unet_config".
"""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from motionclone_b200.synthetic import UNET_SD15_POOLED_GN_CONFIG, UNET_TINY_POOLED_GN_CONFIG  # noqa: E402
from oracle import gen_golden  # noqa: E402
from oracle.gen_golden import BASE, ROOT  # noqa: E402

CASES = {
    # name: (unet width name, inference cfg, input seed), as oracle/gen_golden.py's CASES
    "tiny8_pooledgn": ("tiny", dict(BASE, inference_steps=6, guidance_steps=3, guidance_scale=0.3, video_length=8,
                                    height=128, width=128), 122),
    # 12 frames: also a ragged temporal-attention tile
    "tiny12_pooledgn": ("tiny", dict(BASE, inference_steps=5, guidance_steps=3, guidance_scale=0.4, video_length=12,
                                     height=128, width=128, warm_up_steps=2, cool_up_steps=2), 132),
    "c2mini_pooledgn": ("sd15", dict(BASE, inference_steps=4, guidance_steps=2, guidance_scale=0.4, video_length=16,
                                     height=128, width=128, warm_up_steps=2, cool_up_steps=2), 142),
}
CONFIG_NAMES = {"tiny": "UNET_TINY_POOLED_GN_CONFIG", "sd15": "UNET_SD15_POOLED_GN_CONFIG"}

if __name__ == "__main__":
    names = sys.argv[1:] or list(CASES)
    unknown = [n for n in names if n not in CASES]
    if unknown:
        raise SystemExit(f"unknown case(s) {unknown}; choose from {list(CASES)}")
    gen_golden.CASES.update(CASES)
    gen_golden.UNET_TINY_CONFIG, gen_golden.UNET_SD15_CONFIG = UNET_TINY_POOLED_GN_CONFIG, UNET_SD15_POOLED_GN_CONFIG
    gen_golden.main(names)
    for name in names:  # record which config the fixture was made with (meta is not compared on regeneration)
        path = os.path.join(ROOT, "tests", "golden", f"ref_{name}.npz")
        with np.load(path) as g:
            arrays = {k: g[k] for k in g.files}
        meta = json.loads(str(arrays["meta"]))
        meta.update(unet_config=CONFIG_NAMES[meta["unet"]], generator="scripts/gen_golden_pooled_groupnorm.py")
        arrays["meta"] = np.array(json.dumps(meta))
        np.savez_compressed(path, **arrays)
