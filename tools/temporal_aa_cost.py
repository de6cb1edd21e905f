"""Cost of temporal anti-aliasing (ST_OPT_TEMPORAL_AA) on the GPU: the P_COMPOSITION slot (k_composition with the option off,
k_taa_resolve with it on) on scenes.cornell and scenes.dungeon at 1920x1080, product-tier defaults, both engines in one process,
alternated over several rounds after a warm-up.  Prints the GPU's name and power limit, per scene the median per-frame time of the
slot with its p10-p90 spread (st_pass_times), the median frame time (device events around tick + render), and the achieved bytes
per second against the byte model below.

Byte model (per pixel, float4 = 16 B): the composition reads the G-buffer d0 and d1, the DI and GI diffuse signals and the DI and GI
specular samples (6 x 16 B) and writes `output` (16 B): 112 B.  The resolve reads the same 96 B for its tile plus a 1-pixel halo
(34 x 10 pixels per 32 x 8 tile: x 1.33), the velocity map (16 B), the history's count texel and 16 Catmull-Rom taps (mostly L1 / L2
hits: counted once, 16 B) and writes the history and `output` (32 B): about 96 x 1.33 + 16 + 16 + 32 = 192 B.

    python tools/temporal_aa_cost.py [--rounds 6] [--frames 24] [--size 1920x1080] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import strolle_b200
from strolle_b200 import scenes
from strolle_b200.engine import OPT_TEMPORAL_AA, STAT_TAA_RESOLVES

BYTES_PER_PIXEL = {"off": 112.0, "on": 96.0 * (34 * 10) / (32 * 8) + 16 + 16 + 32}


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def measure(scene, a, w, h):
    engines = {}
    for on in (0, 1):
        e = strolle_b200.Engine()
        e.set_option(OPT_TEMPORAL_AA, on)
        engines[on] = (e, scenes.apply(e, scene))
    for e, cam in engines.values():   # warm-up: both GI cycles' frame shapes, module loads
        for _ in range(12):
            e.tick(); e.render_camera(cam)
        e.synchronize()
        e.enable_timing(True); e.pass_times(reset=True)
    slot = list(strolle_b200.PASS_NAMES).index("frame_composition")
    comp_ms, frame_ms = {0: [], 1: []}, {0: [], 1: []}
    for r in range(a.rounds):
        for on in ((0, 1) if r % 2 == 0 else (1, 0)):
            e, cam = engines[on]
            for _ in range(a.frames):
                e.mark_begin(); e.tick(); e.render_camera(cam)
                frame_ms[on].append(e.mark_end())
                ms, launches = e.pass_times(reset=True)
                comp_ms[on].append(float(ms[slot]) / max(int(launches[slot]), 1))
    for e, _ in engines.values():
        e.enable_timing(False)
    key = lambda k: "on" if k else "off"
    res = dict(median_composition_slot_ms={key(k): round(float(np.median(v)), 5) for k, v in comp_ms.items()},
               p10_p90_composition_slot_ms={key(k): [round(float(np.percentile(v, p)), 5) for p in (10, 90)] for k, v in comp_ms.items()},
               median_frame_ms={key(k): round(float(np.median(v)), 4) for k, v in frame_ms.items()},
               resolves=engines[1][0].get_stat(STAT_TAA_RESOLVES))
    res["achieved_GB_per_s"] = {key(k): round(BYTES_PER_PIXEL[key(k)] * w * h / (float(np.median(v)) * 1e-3) / 1e9, 1) for k, v in comp_ms.items()}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--frames", type=int, default=24)
    ap.add_argument("--size", default="1920x1080")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    w, h = (int(v) for v in a.size.split("x"))
    res = dict(gpu=gpu_info(), size=f"{w}x{h}", rounds=a.rounds, frames_per_round=a.frames, byte_model_per_pixel=BYTES_PER_PIXEL, scenes={})
    for name in ("cornell", "dungeon"):
        res["scenes"][name] = measure(getattr(scenes, name)(w, h), a, w, h)
    print(json.dumps(res, indent=1))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
