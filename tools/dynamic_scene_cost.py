"""Cost of a moving scene with and without ST_OPT_BVH_REFIT: the dungeon with its tori turning (scenes.demo_level_animated) and
scenes.stress_bvh with every object moving, at 1920x1080.  Each frame re-inserts the moved instances, ticks and renders with the frame
copied to the host (RGBA8).  The option off and on (one budget) run in one process, alternated over several rounds.  Prints per
setting: the median wall time per frame and its 10th / 90th percentiles, the median host time of st_tick, the device time of one tick
on an idle stream (st_mark_begin / st_mark_end: the bake + refit launches and their copies with the option on, the uploads without),
Mrays/s, and the mean BVH-heat-map `used_memory` of primary rays after `budget` refit ticks against a fresh rebuild of the same scene.

    python tools/dynamic_scene_cost.py [--rounds 4] [--frames 30] [--budget 30] [--objects 1500] [--size 1920x1080] [--json out.json]
"""
import argparse
import json
import math
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import strolle_b200
from strolle_b200 import scenes
from strolle_b200.engine import FORMAT_RGBA8_SRGB, OPT_BVH_REFIT, STAT_BVH_REFITS
from tools.normal_map_cost import gpu_info


def primary_rays(scene, w, h):
    m = np.asarray(scene["camera"]["transform"], np.float32).reshape(4, 4)
    ys, xs = np.mgrid[0:h, 0:w]
    ndc = np.stack([(xs + 0.5) / w * 2 - 1, 1 - (ys + 0.5) / h * 2], -1).reshape(-1, 2)
    tan = math.tan(math.pi / 8)
    d = (ndc[:, :1] * tan * (w / h)) * m[0, :3] + (ndc[:, 1:] * tan) * m[1, :3] - m[2, :3]
    rays = np.zeros((len(d), 8), np.float32)
    rays[:, 0:3] = m[3, :3]; rays[:, 3] = np.float32(3.4028234663852886e38)
    rays[:, 4:7] = d / np.linalg.norm(d, axis=1, keepdims=True)
    return rays


def workload(name, a):
    w, h = (int(v) for v in a.size.split("x"))
    if name == "dungeon":
        return scenes.demo_level(w, h), lambda t: scenes.demo_level_animated(t)
    return scenes.stress_bvh(a.objects, w, h), lambda t: scenes.stress_bvh_instances(a.objects, t)


def measure(name, a):
    scene, moves = workload(name, a)
    w, h = scene["camera"]["w"], scene["camera"]["h"]
    engines = {}
    for budget in (0, a.budget):
        e = strolle_b200.Engine()
        e.set_option(OPT_BVH_REFIT, budget)
        e.count_rays(True)
        engines[budget] = [e, scenes.apply(e, scene), 0.0]   # engine, camera, scene time
    out = np.zeros((h, w, 4), np.uint8)

    def frame(k):
        e, cam, t = engines[k]
        engines[k][2] = t + 1.0 / 60.0
        for inst in moves(engines[k][2]):
            e.insert_instance(*inst)
        t0 = time.perf_counter()
        e.tick()
        t1 = time.perf_counter()
        e.render_camera(cam, out, FORMAT_RGBA8_SRGB)
        return time.perf_counter() - t0, t1 - t0

    for k in engines:   # warm-up: both GI cycles' frame shapes, module loads
        for _ in range(12):
            frame(k)
    wall, tick = {k: [] for k in engines}, {k: [] for k in engines}
    rays = {k: 0 for k in engines}
    for r in range(a.rounds):
        for k in (sorted(engines) if r % 2 == 0 else sorted(engines, reverse=True)):
            engines[k][0].ray_count(reset=True)
            for _ in range(a.frames):
                fw, ft = frame(k)
                wall[k].append(fw); tick[k].append(ft)
            rays[k] += engines[k][0].ray_count(reset=True)
    device = {}
    for k, (e, cam, t) in engines.items():   # one tick on an idle stream
        samples = []
        for _ in range(5):
            e.synchronize()
            for inst in moves(engines[k][2] + 1.0 / 60.0):
                e.insert_instance(*inst)
            engines[k][2] += 1.0 / 60.0
            before = e.get_stat(STAT_BVH_REFITS)
            e.mark_begin(); e.tick(); ms = e.mark_end()
            if k == 0 or e.get_stat(STAT_BVH_REFITS) > before:
                samples.append(ms)
            e.render_camera(cam, out, FORMAT_RGBA8_SRGB)
        device[k] = round(float(np.median(samples)), 4) if samples else None
    # tree quality: `budget` refit ticks after a rebuild against a rebuild of the same instants
    fresh = {}
    for k in (0, a.budget):
        e = strolle_b200.Engine()
        e.set_option(OPT_BVH_REFIT, k)
        scenes.apply(e, scene)
        e.tick()
        for i in range(a.budget):
            for inst in moves(1.0 + i / 60.0):
                e.insert_instance(*inst)
            e.tick()
        fresh[k] = (e, e.get_stat(STAT_BVH_REFITS))
    pr = primary_rays(scene, w // 4, h // 4)
    used = {k: float(fresh[k][0].trace_closest(pr).reshape(-1, 12)[:, 11].astype(np.float64).mean()) for k in fresh}
    label = lambda k: "off" if k == 0 else f"on_{k}"
    total = {k: float(np.sum(wall[k])) for k in wall}
    return dict(scene=name, size=f"{w}x{h}", instances=len(scene["instances"]), rounds=a.rounds, frames_per_round=a.frames,
                median_frame_ms={label(k): round(1e3 * float(np.median(v)), 4) for k, v in wall.items()},
                p10_p90_frame_ms={label(k): [round(1e3 * float(np.percentile(v, p)), 4) for p in (10, 90)] for k, v in wall.items()},
                median_tick_host_ms={label(k): round(1e3 * float(np.median(v)), 4) for k, v in tick.items()},
                tick_device_ms={label(k): v for k, v in device.items()},
                mrays_per_s={label(k): round(rays[k] / total[k] / 1e6, 1) for k in rays},
                refit_ticks={label(k): engines[k][0].get_stat(STAT_BVH_REFITS) for k in engines},
                heatmap_used_memory_mean={"rebuild": round(used[0], 3), f"after_{fresh[a.budget][1]}_refits": round(used[a.budget], 3)})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--frames", type=int, default=30)
    ap.add_argument("--budget", type=int, default=30)
    ap.add_argument("--objects", type=int, default=1500)
    ap.add_argument("--size", default="1920x1080")
    ap.add_argument("--scenes", default="dungeon,stress")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    res = dict(gpu=gpu_info(), results=[measure(s, a) for s in a.scenes.split(",")])
    print(json.dumps(res, indent=1))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
