"""Cost of environment-map sampling (ST_OPT_ENVIRONMENT_MAP_SAMPLING) on the GPU, in one process: the distribution build for
2048x1024 and 8192x4096 maps (device events around the tick that builds it, less a plain tick); per scene (env_courtyard,
env_sunlit at 1920x1080, product-tier defaults) the median frame time with its p10-p90 spread with the option off and on, alternated
over several rounds, and the per-frame device time of gi_sampling_a / gi_sampling_b (st_pass_times, separate frames); and the noise
ratio: the per-pixel variance of the composed frame's luminance (denoising off) over 64 frames, off over on.  Prints the GPU's name
and power limit.

    python tools/environment_map_sampling_cost.py [--rounds 6] [--frames 24] [--size 1920x1080] [--json out.json]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import strolle_b200
from strolle_b200 import scenes
from strolle_b200.engine import OPT_ENVIRONMENT_MAP_SAMPLING, STAT_ENVIRONMENT_MAP_DISTRIBUTION_BUILDS
from tools.environment_map_cost import gpu_info

LUMA = np.array([0.2126, 0.7152, 0.0722])


def build_ms(size, a):
    """Median device time of the tick that builds a size[0] x size[1] map's distribution, less the median plain tick."""
    w, h = size
    sky = scenes.sunlit_sky(w, h)
    e = strolle_b200.Engine()
    scenes.apply(e, scenes.env_sunlit(64, 36))
    e.set_option(OPT_ENVIRONMENT_MAP_SAMPLING, 1)
    e.set_environment_map(sky, 1.0, 0.0); e.tick(); e.synchronize()
    build, plain = [], []
    for _ in range(a.builds):
        e.set_option(OPT_ENVIRONMENT_MAP_SAMPLING, 0); e.tick()
        e.set_option(OPT_ENVIRONMENT_MAP_SAMPLING, 1)
        e.mark_begin(); e.tick(); build.append(e.mark_end())
        e.mark_begin(); e.tick(); plain.append(e.mark_end())
    assert e.get_stat(STAT_ENVIRONMENT_MAP_DISTRIBUTION_BUILDS) == a.builds + 1
    return round(float(np.median(build) - np.median(plain)), 4)


def measure(scene, a):
    engines = {}
    for on in (0, 1):
        e = strolle_b200.Engine()
        cam = scenes.apply(e, scene)
        e.set_option(OPT_ENVIRONMENT_MAP_SAMPLING, on)
        engines[on] = (e, cam)
    for e, cam in engines.values():
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
        passes[on] = {n: round(float(ms[i]) / a.frames, 4) for i, n in enumerate(names) if launches[i] and "gi_sampling" in n}
    noise = {}
    for on in (0, 1):   # per-pixel variance of the composed luminance, denoising off
        sc = dict(scene); sc["camera"] = dict(scene["camera"], denoise=False)
        e = strolle_b200.Engine(); cam = scenes.apply(e, sc); e.set_option(OPT_ENVIRONMENT_MAP_SAMPLING, on)
        s1 = s2 = 0.0
        for _ in range(a.noise_frames):
            e.tick(); e.render_camera(cam)
            y = e.read_buffer(cam, "output").reshape(-1, 4)[:, :3].astype(np.float64) @ LUMA
            s1, s2 = s1 + y, s2 + y * y
        m = s1 / a.noise_frames
        noise[on] = (float(m.mean()), float((s2 / a.noise_frames - m * m).mean()))
    key = lambda k: "on" if k else "off"
    return dict(median_frame_ms={key(k): round(float(np.median(v)), 4) for k, v in frame_ms.items()},
                p10_p90_frame_ms={key(k): [round(float(np.percentile(v, p)), 4) for p in (10, 90)] for k, v in frame_ms.items()},
                pass_ms_per_frame={key(k): v for k, v in passes.items()},
                mean_luminance={key(k): round(v[0], 5) for k, v in noise.items()},
                pixel_variance={key(k): v[1] for k, v in noise.items()}, noise_ratio_off_over_on=round(noise[0][1] / noise[1][1], 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--frames", type=int, default=24)
    ap.add_argument("--builds", type=int, default=9)
    ap.add_argument("--noise-frames", type=int, default=64)
    ap.add_argument("--size", default="1920x1080")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    w, h = (int(v) for v in a.size.split("x"))
    res = dict(gpu=gpu_info(), size=f"{w}x{h}", rounds=a.rounds, frames_per_round=a.frames,
               build_ms={f"{bw}x{bh}": build_ms((bw, bh), a) for bw, bh in ((2048, 1024), (8192, 4096))}, scenes={})
    for name in ("env_courtyard", "env_sunlit"):
        res["scenes"][name] = measure(getattr(scenes, name)(w, h), a)
    print(json.dumps(res, indent=1))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
