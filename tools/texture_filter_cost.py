"""Cost of texture filtering (ST_OPT_TEXTURE_FILTER) on the GPU: scenes.demo_level and scenes.tiled_ground at 1920x1080, the option
off and on, in one process, alternated over several rounds.  Prints the GPU's name and power limit, per scene the median frame time
of each with its p10-p90 spread (device events around tick + render, product-tier defaults), the per-frame device time of the G-buffer
pass and of GI sampling (st_pass_times, timed in separate frames), and the time of a tick that rebuilds the mip chains.

    python tools/texture_filter_cost.py [--rounds 6] [--frames 24] [--size 1920x1080] [--json out.json]
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
from strolle_b200.engine import OPT_TEXTURE_FILTER, STAT_TEXTURE_MIP_BUILDS


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def measure(scene, a):
    engines = {}
    for on in (0, 1):
        e = strolle_b200.Engine()
        e.set_option(OPT_TEXTURE_FILTER, on)
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
    e, cam = engines[1]   # ticks that rebuild the chains (the option turned off, then on), against plain ticks
    build_ms, plain_ms = [], []
    for _ in range(a.frames):
        e.set_option(OPT_TEXTURE_FILTER, 0); e.tick(); e.set_option(OPT_TEXTURE_FILTER, 1)
        e.mark_begin(); e.tick(); build_ms.append(e.mark_end())
        e.mark_begin(); e.tick(); plain_ms.append(e.mark_end())
    return dict(median_frame_ms={("on" if k else "off"): round(float(np.median(v)), 4) for k, v in frame_ms.items()},
                p10_p90_frame_ms={("on" if k else "off"): [round(float(np.percentile(v, p)), 4) for p in (10, 90)] for k, v in frame_ms.items()},
                pass_ms_per_frame={("on" if k else "off"): v for k, v in passes.items()},
                mip_build_tick_ms=round(float(np.median(build_ms)), 4), plain_tick_ms=round(float(np.median(plain_ms)), 4),
                mip_builds=e.get_stat(STAT_TEXTURE_MIP_BUILDS))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--frames", type=int, default=24)
    ap.add_argument("--size", default="1920x1080")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    w, h = (int(v) for v in a.size.split("x"))
    res = dict(gpu=gpu_info(), size=f"{w}x{h}", rounds=a.rounds, frames_per_round=a.frames, scenes={})
    for name in ("demo_level", "tiled_ground"):
        res["scenes"][name] = measure(getattr(scenes, name)(w, h), a)
    print(json.dumps(res, indent=1))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
