"""Cost of the environment map (st_set_environment_map) on the GPU: scenes.env_courtyard and scenes.tiled_ground at 1920x1080, with no
map and with a 2048x1024 map (scenes.courtyard_sky), in one process, alternated over several rounds.  Prints the GPU's name and power
limit, per scene the median frame time of each with its p10-p90 spread (device events around tick + render, product-tier defaults),
the per-frame device time of di_resolving and of GI sampling (st_pass_times, timed in separate frames), and the cost of setting a map:
the host time of st_set_environment_map (validation and copy) and the device-event time of the tick that uploads it, against a plain
tick.

    python tools/environment_map_cost.py [--rounds 6] [--frames 24] [--size 1920x1080] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import strolle_b200
from strolle_b200 import scenes
from strolle_b200.engine import STAT_ENVIRONMENT_MAP_LAUNCHES


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def measure(scene, sky, a):
    scene = dict(scene)
    scene.pop("environment_map", None)
    engines = {}
    for on in (0, 1):
        e = strolle_b200.Engine()
        cam = scenes.apply(e, scene)
        if on:
            e.set_environment_map(sky, 1.5, 0.0)
        engines[on] = (e, cam)
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
        passes[on] = {n: round(float(ms[i]) / a.frames, 4) for i, n in enumerate(names) if launches[i] and ("di_resolving" in n or "gi_sampling" in n)}
    e, cam = engines[1]   # setting a map: the call on the host, then the tick that uploads it, against a plain tick
    set_ms, upload_ms, plain_ms = [], [], []
    for _ in range(a.frames):
        e.synchronize()
        t0 = time.perf_counter(); e.set_environment_map(sky, 1.5, 0.0); set_ms.append((time.perf_counter() - t0) * 1e3)
        e.mark_begin(); e.tick(); upload_ms.append(e.mark_end())
        e.mark_begin(); e.tick(); plain_ms.append(e.mark_end())
    return dict(median_frame_ms={("map" if k else "none"): round(float(np.median(v)), 4) for k, v in frame_ms.items()},
                p10_p90_frame_ms={("map" if k else "none"): [round(float(np.percentile(v, p)), 4) for p in (10, 90)] for k, v in frame_ms.items()},
                pass_ms_per_frame={("map" if k else "none"): v for k, v in passes.items()},
                set_call_host_ms=round(float(np.median(set_ms)), 4), upload_tick_ms=round(float(np.median(upload_ms)), 4),
                plain_tick_ms=round(float(np.median(plain_ms)), 4), envm_launches=e.get_stat(STAT_ENVIRONMENT_MAP_LAUNCHES))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--frames", type=int, default=24)
    ap.add_argument("--size", default="1920x1080")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    w, h = (int(v) for v in a.size.split("x"))
    sky = scenes.courtyard_sky(2048, 1024)
    res = dict(gpu=gpu_info(), size=f"{w}x{h}", map="2048x1024 float4 (32 MiB)", rounds=a.rounds, frames_per_round=a.frames, scenes={})
    for name in ("env_courtyard", "tiled_ground"):
        res["scenes"][name] = measure(getattr(scenes, name)(w, h), sky, a)
    print(json.dumps(res, indent=1))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
