"""Cost of depth of field (ST_OPT_DEPTH_OF_FIELD) on the GPU: scenes.cornell, scenes.dungeon and scenes.env_sunlit at 1920x1080,
product-tier defaults, with the option off and on at max_radius 8, 16 and 32, the engines alternated over several rounds after a warm-up.
The lens focuses at the median view depth of the first frame with k = 2 R (the CoC at infinity twice the clamp), so that most tiles
gather at or near the largest radius: a heavy case, not a typical one.  Each frame is rendered and copied out as Rgba32F.  Prints the
GPU's name and power limit, per scene and radius the median P_COMPOSITION slot per frame (the composition, the CoC and the gather are
all timed there) with its p10-p90 spread, and, from a torch.profiler run of its own, the median device time of k_dof_coc and
k_dof_gather per frame.

    python tools/depth_of_field_cost.py [--rounds 4] [--frames 12] [--size 1920x1080] [--json out.json]
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
from strolle_b200.engine import FORMAT_RGBA32F, OPT_DEPTH_OF_FIELD, STAT_DEPTH_OF_FIELD_GATHERS

SENSOR = 0.01866


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def lens(e, cam, scene, R):
    """Focus at the median view depth of the camera's current frame, k = 2 R."""
    w, h = scene["camera"]["w"], scene["camera"]["h"]
    t = e.read_buffer(cam, "surface_nd").reshape(h, w, 4)[..., 3]
    F = float(np.median(t[t > 0])) if (t > 0).any() else 5.0
    f = 0.5 * SENSOR * float(scene["camera"]["projection"][5])
    N = f * f / (F - f) * h / SENSOR / 2.0 / (2.0 * R)
    return dict(focal_distance=F, aperture_f_stops=N, sensor_height=SENSOR, max_radius=float(R))


def engine(scene, R):
    """An engine with the option on (R > 0) or off (R = 0), warmed up over both GI cycles' frame shapes."""
    w, h = scene["camera"]["w"], scene["camera"]["h"]
    e = strolle_b200.Engine()
    cam = scenes.apply(e, scene)
    e.tick(); e.render_camera(cam)
    if R:
        e.set_option(OPT_DEPTH_OF_FIELD, 1)
        e.set_depth_of_field(**lens(e, cam, scene, R))
    host = np.zeros((h, w, 4), np.float32)
    for _ in range(12):
        e.tick(); e.render_camera(cam, host, FORMAT_RGBA32F)
    e.synchronize()
    return e, cam, host


def measure(scene, a, radii):
    engines = {R: engine(scene, R) for R in (0,) + radii}
    for e, _, _ in engines.values():
        e.enable_timing(True); e.pass_times(reset=True)
    slot = list(strolle_b200.PASS_NAMES).index("frame_composition")
    comp = {R: [] for R in engines}
    order = list(engines)
    for r in range(a.rounds):
        for R in (order if r % 2 == 0 else order[::-1]):
            e, cam, host = engines[R]
            for _ in range(a.frames):
                e.tick(); e.render_camera(cam, host, FORMAT_RGBA32F)
                ms, _ = e.pass_times(reset=True)
                comp[R].append(float(ms[slot]))
    for e, _, _ in engines.values():
        e.enable_timing(False)
    q = lambda v: [round(float(np.percentile(v, p)), 4) for p in (50, 10, 90)]
    res = {"off" if R == 0 else f"R{R}": dict(composition_slot_ms_p50_p10_p90=q(v)) for R, v in comp.items()}
    base = float(np.median(comp[0]))
    for R in radii:
        res[f"R{R}"]["slot_growth_ms"] = round(float(np.median(comp[R])) - base, 4)
        res[f"R{R}"]["gathers"] = engines[R][0].get_stat(STAT_DEPTH_OF_FIELD_GATHERS)
    return res


def kernel_times(scene, R, frames=12):
    """Median device time per frame of k_dof_coc and k_dof_gather, from torch.profiler (CUDA activities)."""
    from torch.profiler import ProfilerActivity, profile
    e, cam, host = engine(scene, R)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(frames):
            e.tick(); e.render_camera(cam, host, FORMAT_RGBA32F)
        e.synchronize()
    times = {}
    for ev in prof.events():
        for tag in ("k_dof_coc", "k_dof_gather"):
            if tag in ev.name and ev.device_type.name == "CUDA":
                times.setdefault(tag, []).append(ev.device_time_total)
    return {k: round(float(np.median(v)), 2) for k, v in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--frames", type=int, default=12)
    ap.add_argument("--size", default="1920x1080")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    w, h = (int(v) for v in a.size.split("x"))
    radii = (8, 16, 32)
    res = dict(gpu=gpu_info(), size=f"{w}x{h}", rounds=a.rounds, frames_per_round=a.frames, scenes={})
    for name in ("cornell", "dungeon", "env_sunlit"):
        sc = getattr(scenes, name)(w, h)
        res["scenes"][name] = measure(sc, a, radii)
        for R in radii:
            res["scenes"][name][f"R{R}"]["kernel_us"] = kernel_times(sc, R)
    print(json.dumps(res, indent=1))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
