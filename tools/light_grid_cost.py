"""Cost and benefit of the light grid (ST_OPT_LIGHT_GRID) on the GPU: scenes.stress_lights with the lights animated every tick, the
option off and on (N = 32) in one process, alternated over several rounds, product-tier defaults.  Prints the GPU's name and power
limit and, per size: the median frame and its p10-p90 spread (device events around tick + render), the build's device time per tick
(a tick whose only change is N, so the build is all it enqueues), the per-frame device time of the fused DI sampling launch and of
the GI sampling launch (st_pass_times), the Reference-mode variance ratio and the ReSTIR DI single-frame noise, on against off; then
the build time at 100, 1,000 and 10,000 lights with N = 32.

    python tools/light_grid_cost.py [--rounds 6] [--frames 24] [--sizes 1920x1080,512x512] [--json out.json]
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
from strolle_b200.engine import OPT_LIGHT_GRID, STAT_LIGHT_GRID_BUILDS

N = 32


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def animate(e, t):
    for h, kind, params in scenes.stress_lights_lights(t):
        e.insert_light(h, kind, params)


def build_ms(e, ticks=20):
    """Device time of a tick that only rebuilds the grid (N toggled between 32 and 31), median."""
    out = []
    for k in range(ticks):
        e.set_option(OPT_LIGHT_GRID, N if k % 2 == 0 else N - 1)
        e.mark_begin(); e.tick(); out.append(e.mark_end())
    e.set_option(OPT_LIGHT_GRID, N); e.tick()
    return float(np.median(out))


def frame_costs(w, h, rounds, frames):
    scene = scenes.stress_lights(w, h)
    engines = {}
    for n in (0, N):
        e = strolle_b200.Engine()
        e.set_option(OPT_LIGHT_GRID, n)
        engines[n] = (e, scenes.apply(e, scene))
    t = 0.0
    for e, cam in engines.values():   # warm-up: both GI cycles' frame shapes, module loads
        for k in range(12):
            animate(e, 0.02 * k); e.tick(); e.render_camera(cam)
        e.synchronize()
    frame_ms = {0: [], N: []}
    for r in range(rounds):
        for n in ((0, N) if r % 2 == 0 else (N, 0)):
            e, cam = engines[n]
            for k in range(frames):
                t += 0.016
                animate(e, t)
                e.mark_begin(); e.tick(); e.render_camera(cam)
                frame_ms[n].append(e.mark_end())
    names = list(strolle_b200.PASS_NAMES)
    passes = {}
    for n, (e, cam) in engines.items():
        e.enable_timing(True); e.pass_times(reset=True)
        for k in range(frames):
            animate(e, t + 0.016 * k); e.tick(); e.render_camera(cam)
        e.synchronize()
        ms, launches = e.pass_times(reset=True)
        e.enable_timing(False)
        passes[n] = {nm: round(float(ms[i]) / frames, 4) for i, nm in enumerate(names) if launches[i] and ("di_temporal" in nm or "gi_sampling" in nm)}
    key = lambda n: "on" if n else "off"
    return dict(median_frame_ms={key(n): round(float(np.median(v)), 4) for n, v in frame_ms.items()},
                p10_p90_frame_ms={key(n): [round(float(np.percentile(v, p)), 4) for p in (10, 90)] for n, v in frame_ms.items()},
                pass_ms_per_frame={key(n): v for n, v in passes.items()},
                build_ms_per_tick=round(build_ms(engines[N][0]), 4),
                builds=engines[N][0].get_stat(STAT_LIGHT_GRID_BUILDS))


def noise(w=128, h=128, frames=128):
    """Reference mode (depth 1) per-pixel variance ratio on / off, and ReSTIR DI (MODE_DI_DIFFUSE, no denoiser) single-frame
    relative L2 against the frame mean, static lights."""
    out = {}
    ref = scenes.stress_lights(w, h, mode=scenes.MODE_REFERENCE, ref_depth=1, t=0.3)
    var = {}
    for n in (0, N):
        e = strolle_b200.Engine(); e.set_option(OPT_LIGHT_GRID, n)
        cam = scenes.apply(e, ref)
        prev, fr = np.zeros((h, w)), []
        for _ in range(frames):
            e.tick(); e.render_camera(cam)
            acc = e.read_buffer(cam, "ref_colors").reshape(h, w, 4)[..., :3].astype(np.float64).sum(-1)
            fr.append(acc - prev); prev = acc
        var[n] = float(np.var(fr, 0).mean())
    out["reference_variance_ratio_on_off"] = round(var[N] / var[0], 4)
    di = scenes.stress_lights(w, h, mode=scenes.MODE_DI_DIFFUSE, denoise=False, t=0.3)
    l2 = {}
    for n in (0, N):
        e = strolle_b200.Engine(); e.set_option(OPT_LIGHT_GRID, n)
        cam = scenes.apply(e, di)
        fr = []
        for _ in range(2 * frames):
            e.tick(); e.render_camera(cam)
            fr.append(e.read_buffer(cam, "output").reshape(h, w, 4)[..., :3].astype(np.float64))
        mean = np.mean(fr, 0)
        l2[n] = float(np.mean([np.linalg.norm(fr[k] - mean) / np.linalg.norm(mean) for k in (frames // 2, frames, 3 * frames // 2)]))
    out["restir_di_rel_l2"] = {"on": round(l2[N], 4), "off": round(l2[0], 4)}
    return out


def build_scaling():
    """Build time per tick at 100, 1,000 and 10,000 random point lights of range 20 over a 150 x 150 x 20 region, N = 32."""
    out = {}
    rng = np.random.RandomState(3)
    for count in (100, 1000, 10000):
        e = strolle_b200.Engine(); e.set_option(OPT_LIGHT_GRID, N)
        sc = scenes.stress_lights(64, 64)
        sc = dict(sc, lights=[(1000 + k, scenes.LIGHT_POINT, scenes.point_light(tuple(rng.uniform((-75, 0, -10), (75, 150, 10))), 0.25,
                                                                                  (1.0, 1.0, 1.0), 20.0)) for k in range(count)])
        scenes.apply(e, sc)
        e.tick(); e.synchronize()
        out[count] = round(build_ms(e), 4)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--frames", type=int, default=24)
    ap.add_argument("--sizes", default="1920x1080,512x512")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    res = dict(gpu=gpu_info(), n=N, rounds=a.rounds, frames_per_round=a.frames, sizes={})
    for s in a.sizes.split(","):
        w, h = (int(v) for v in s.split("x"))
        res["sizes"][s] = frame_costs(w, h, a.rounds, a.frames)
        print(s, json.dumps(res["sizes"][s]), flush=True)
    res["noise_128x128"] = noise()
    res["build_ms_by_lights"] = build_scaling()
    print(json.dumps(res, indent=1))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
