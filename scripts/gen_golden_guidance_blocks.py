"""Generates the guidance-block fixtures tests/golden/ref_{tiny8_up12,tiny4_all40,tiny8_midv2,c2mini8_up3}.npz by running
the UNMODIFIED reference on the CPU with other `motion_guidance_blocks` than the shipped ['up_blocks.1'], through
oracle/gen_golden.py's writer (same inputs, same checks: regenerating must reproduce every committed tensor bit for bit).
TEST INFRASTRUCTURE: needs the reference tree, like oracle/gen_golden.py.

  python scripts/gen_golden_guidance_blocks.py [tiny8_up12 tiny4_all40 tiny8_midv2 c2mini8_up3]

The writer picks the UNet config by the names "tiny" / "sd15". The mid-block case runs the tiny widths with
motion_module_mid_block=True (configs/model_config/inference-v2.yaml); it is written under the name "tiny_midv2" with the
"sd15" slot pointing at that config, so the writer does not overwrite the plain tiny state-dict shapes. The config name
is recorded in each fixture's meta as "unet_config".

Every fixture stays under MAX_BYTES. The motion representation (fp32 top-1 values, incompressible) is most of a
fixture, and it grows with the guided modules' positions x heads x frames: with 40 modules, or 6 modules at the
full-resolution level, 8 frames would exceed the bound, so those two cases run 4 frames (tiny4_all40; a ragged clip
length) and 8 frames (c2mini8_up3, SD1.5 widths). Besides, the full extraction probabilities are dropped, as for c1;
top-2 probability gaps at or above NEAR_TIE (the bound the GPU tests hold index mismatches to) are stored as 1.0, since
only gaps below it are ever read; and those two cases keep the latents of the first step, the last guided step, the
first plain step and the end only (KEEP_STEPS). The regeneration check of oracle/gen_golden.py (GOLDEN_CHECK_STABLE, on
by default) runs here on the written arrays.
"""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from motionclone_b200.synthetic import UNET_SD15_CONFIG, UNET_TINY_CONFIG, UNET_TINY_MIDV2_CONFIG  # noqa: E402
from oracle import gen_golden  # noqa: E402
from oracle.gen_golden import BASE, ROOT  # noqa: E402

UP = ["up_blocks.0", "up_blocks.1", "up_blocks.2", "up_blocks.3"]
TINY8 = dict(BASE, inference_steps=6, guidance_steps=3, guidance_scale=0.3, video_length=8, height=128, width=128)
CASES = {
    # name: (unet width name, inference cfg, input seed), as oracle/gen_golden.py's CASES
    # two levels (h/32 and h/16), cut 2
    "tiny8_up12": ("tiny", dict(TINY8, motion_guidance_blocks=["up_blocks.1", "up_blocks.2"]), 152),
    # every temporal attention of the UNet (40 modules), so the whole UNet carries gradient
    "tiny4_all40": ("tiny", dict(TINY8, video_length=4, motion_guidance_blocks=["down_blocks"] + UP), 162),
    # the v2 model config's mid-block motion module (2 modules) and up_blocks.1
    "tiny8_midv2": ("tiny_midv2", dict(TINY8, motion_guidance_blocks=["mid_block", "up_blocks.1"]), 172),
    # SD1.5 widths, 8 frames: the full-resolution level (head dim 40), cut 3
    "c2mini8_up3": ("sd15", dict(BASE, inference_steps=4, guidance_steps=2, guidance_scale=0.4, video_length=8,
                                height=128, width=128, warm_up_steps=2, cool_up_steps=2,
                                motion_guidance_blocks=["up_blocks.3"]), 182),
}
NEAR_TIE = 8e-3
KEEP_STEPS = {"tiny4_all40": [0, 2, 3, 5], "c2mini8_up3": [0, 2, 3]}
MAX_BYTES = 950_000
CONFIG_NAMES = {"tiny": "UNET_TINY_CONFIG", "tiny_midv2": "UNET_TINY_MIDV2_CONFIG", "sd15": "UNET_SD15_CONFIG"}

if __name__ == "__main__":
    names = sys.argv[1:] or list(CASES)
    unknown = [n for n in names if n not in CASES]
    if unknown:
        raise SystemExit(f"unknown case(s) {unknown}; choose from {list(CASES)}")
    gen_golden.CASES.update(CASES)
    check_stable = os.environ.get("GOLDEN_CHECK_STABLE", "1") == "1"
    os.environ["GOLDEN_CHECK_STABLE"] = "0"  # the writer's own check would compare before the reductions below
    for name in names:
        gen_golden.UNET_TINY_CONFIG = UNET_TINY_CONFIG
        gen_golden.UNET_SD15_CONFIG = UNET_TINY_MIDV2_CONFIG if CASES[name][0] == "tiny_midv2" else UNET_SD15_CONFIG
        path = os.path.join(ROOT, "tests", "golden", f"ref_{name}.npz")
        old = None
        if check_stable and os.path.exists(path):
            with np.load(path) as g:
                old = {k: g[k] for k in g.files}
        gen_golden.main([name])
        with np.load(path) as g:
            arrays = {k: g[k] for k in g.files}
        arrays.pop("extract_probs_0", None)
        for k in arrays:
            if k.startswith("extract_top2gap_"):
                arrays[k] = np.where(arrays[k] < NEAR_TIE, arrays[k], np.float32(1.0)).astype(np.float32)
        if name in KEEP_STEPS:
            arrays["latents_per_step"] = arrays["latents_per_step"][KEEP_STEPS[name]]
            arrays["latents_steps_kept"] = np.array(KEEP_STEPS[name])
        if old is not None:  # regenerating must reproduce every tensor already committed, bit for bit
            for k in old:
                if k != "meta":
                    assert np.array_equal(old[k], arrays[k]), f"{name}: regenerated '{k}' differs from the committed fixture"
        meta = json.loads(str(arrays["meta"]))  # meta is not compared on regeneration
        meta.update(unet_config=CONFIG_NAMES[meta["unet"]], generator="scripts/gen_golden_guidance_blocks.py")
        arrays["meta"] = np.array(json.dumps(meta))
        np.savez_compressed(path, **arrays)
        assert os.path.getsize(path) < MAX_BYTES, f"{name}: {os.path.getsize(path)} bytes, the bound is {MAX_BYTES}"
        print(name, "->", os.path.getsize(path) // 1024, "KiB after dropping the full probabilities", flush=True)
