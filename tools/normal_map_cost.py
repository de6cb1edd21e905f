"""Cost of normal mapping (ST_OPT_NORMAL_MAPS) on the GPU: scenes.normal_mapped_room at 1920x1080, the option off and on, in one
process, alternated over several rounds.  Prints the GPU's name and power limit, the median frame time of each (device events around
tick + render, product-tier defaults) and the per-frame device time of the G-buffer pass and of GI sampling (st_pass_times, timed in
separate frames).

    python tools/normal_map_cost.py [--rounds 6] [--frames 24] [--size 1920x1080] [--json out.json]
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
from strolle_b200.engine import OPT_NORMAL_MAPS, STAT_NORMAL_MAP_LAUNCHES


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--frames", type=int, default=24)
    ap.add_argument("--size", default="1920x1080")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    w, h = (int(v) for v in a.size.split("x"))
    scene = scenes.normal_mapped_room(w, h)
    engines = {}
    for on in (0, 1):
        e = strolle_b200.Engine()
        e.set_option(OPT_NORMAL_MAPS, on)
        engines[on] = (e, scenes.apply(e, scene))
    for e, cam in engines.values():   # warm-up: both GI cycles' frame shapes, module loads
        for _ in range(12):
            e.tick(); e.render_camera(cam)
        e.synchronize()
    frame_ms = {0: [], 1: []}
    for r in range(a.rounds):
        for on in ((0, 1) if r % 2 == 0 else (1, 0)):
            e, cam = engines[on]
            for _ in range(a.frames):
                e.mark_begin(); e.tick(); e.render_camera(cam)
                frame_ms[on].append(e.mark_end())
    names = list(strolle_b200.PASS_NAMES)
    passes = {}
    for on, (e, cam) in engines.items():
        e.enable_timing(True); e.pass_times(reset=True)
        for _ in range(a.frames):
            e.tick(); e.render_camera(cam)
        e.synchronize()
        ms, launches = e.pass_times(reset=True)
        e.enable_timing(False)
        passes[on] = {n: round(float(ms[i]) / a.frames, 4) for i, n in enumerate(names) if launches[i] and ("gbuffer" in n or "gi_sampling" in n)}
    res = dict(gpu=gpu_info(), size=f"{w}x{h}", rounds=a.rounds, frames_per_round=a.frames,
               median_frame_ms={("on" if k else "off"): round(float(np.median(v)), 4) for k, v in frame_ms.items()},
               p10_p90_frame_ms={("on" if k else "off"): [round(float(np.percentile(v, p)), 4) for p in (10, 90)] for k, v in frame_ms.items()},
               pass_ms_per_frame={("on" if k else "off"): v for k, v in passes.items()},
               nmap_launches={("on" if k else "off"): engines[k][0].get_stat(STAT_NORMAL_MAP_LAUNCHES) for k in (0, 1)})
    print(json.dumps(res, indent=1))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
