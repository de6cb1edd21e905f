"""Cost of bloom (ST_OPT_BLOOM) on the GPU: scenes.cornell, scenes.dungeon and scenes.env_sunlit at 1920x1080, product-tier defaults
(bloom defaults, L = 7, tonemapping off), with the option off and on, both engines in one process, alternated over several rounds after
a warm-up.  Each frame is rendered and copied out as Rgba8UnormSrgb.  Prints the GPU's name and power limit, per scene and setting the
median frame time (device events around tick + render + copy) with its p10-p90 spread, the P_COMPOSITION slot per frame (the
composition, the pyramid and the Rgba8 store are all timed there) and the Rgba8 st_copy_output device time; then, from a torch.profiler
run of its own, the median kernel times of the pyramid kernels (k_bloom_*), k_output_bloom<0> and k_output_rgba8.

Byte model (bytes_model below): the first downsample reads `output` once (16 B per pixel) and writes level 0; each later level reads its
source level once and writes itself; the up chain reads down_k and up_{k+1} and writes up_k; the store reads up_0 beyond what it reads
with the option off.  Their time at the data sheet's 3.35 TB/s is a floor, not a measurement.

    python tools/bloom_cost.py [--rounds 6] [--frames 16] [--size 1920x1080] [--json out.json]
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
from strolle_b200.engine import BLOOM_DEFAULTS, FORMAT_RGBA8_SRGB, OPT_BLOOM, STAT_BLOOM_PYRAMIDS

HBM_BYTES_PER_S = 3.35e12


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def _engine(scene, on):
    e = strolle_b200.Engine()
    if on:
        e.set_option(OPT_BLOOM, 1)
    return e, scenes.apply(e, scene)


def measure(scene, a, w, h):
    import torch
    host = torch.zeros((h, w, 4), dtype=torch.uint8, pin_memory=True).numpy()
    engines = {on: _engine(scene, on) for on in (0, 1)}
    for e, cam in engines.values():   # warm-up: both GI cycles' frame shapes, module loads
        for _ in range(12):
            e.tick(); e.render_camera(cam, host, FORMAT_RGBA8_SRGB)
        e.synchronize()
        e.enable_timing(True); e.pass_times(reset=True)
    slot = list(strolle_b200.PASS_NAMES).index("frame_composition")
    comp, frame, copy = ({0: [], 1: []} for _ in range(3))
    for r in range(a.rounds):
        for on in ((0, 1) if r % 2 == 0 else (1, 0)):
            e, cam = engines[on]
            for _ in range(a.frames):
                e.mark_begin(); e.tick(); e.render_camera(cam, host, FORMAT_RGBA8_SRGB)
                frame[on].append(e.mark_end())
                ms, _ = e.pass_times(reset=True)
                comp[on].append(float(ms[slot]))
                e.mark_begin(); e.copy_output(cam, host, FORMAT_RGBA8_SRGB)
                copy[on].append(e.mark_end())
                e.pass_times(reset=True)
    for e, _ in engines.values():
        e.enable_timing(False)
    key = lambda k: "bloom" if k else "off"
    q = lambda v: [round(float(np.percentile(v, p)), 4) for p in (50, 10, 90)]
    return dict(frame_ms_p50_p10_p90={key(k): q(v) for k, v in frame.items()},
                composition_slot_ms_p50_p10_p90={key(k): q(v) for k, v in comp.items()},
                rgba8_copy_output_ms_p50_p10_p90={key(k): q(v) for k, v in copy.items()},
                pyramids=engines[1][0].get_stat(STAT_BLOOM_PYRAMIDS))


def kernel_times(scene, w, h, frames=12):
    """Median device time per launch of the display kernels, from torch.profiler (CUDA activities) over `frames` frames."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    host = torch.zeros((h, w, 4), dtype=torch.uint8, pin_memory=True).numpy()
    e, cam = _engine(scene, 1)
    off, coff = _engine(scene, 0)
    for _ in range(6):
        e.tick(); e.render_camera(cam, host, FORMAT_RGBA8_SRGB); off.tick(); off.render_camera(coff, host, FORMAT_RGBA8_SRGB)
    e.synchronize(); off.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(frames):
            e.tick(); e.render_camera(cam, host, FORMAT_RGBA8_SRGB); off.tick(); off.render_camera(coff, host, FORMAT_RGBA8_SRGB)
        e.synchronize(); off.synchronize()
    times = {}
    for ev in prof.events():
        for tag in ("k_bloom_down0", "k_bloom_down", "k_bloom_tail", "k_bloom_up", "k_output_bloom", "k_output_rgba8"):
            if tag == "k_bloom_down" and "k_bloom_down0" in ev.name:
                continue
            if tag in ev.name and ev.device_type.name == "CUDA":
                times.setdefault(tag, []).append(ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total)
    return {k: dict(median_us=round(float(np.median(v)), 2), total_us_per_frame=round(float(np.sum(v)) / frames, 2), launches=len(v))
            for k, v in times.items()}


def bytes_model(w, h, levels=BLOOM_DEFAULTS["levels"]):
    """Bytes the pyramid and the bloomed store move per frame (see the module docstring)."""
    sz = [(max(1, w >> (k + 1)), max(1, h >> (k + 1))) for k in range(levels)]
    n = [a * b for a, b in sz]
    down = 16 * w * h + 16 * n[0] + sum(16 * n[k - 1] + 16 * n[k] for k in range(1, levels))
    up = sum(16 * n[k] + 16 * n[k + 1] + 16 * n[k] for k in range(levels - 1))
    store_extra = 16 * n[0]   # the bloomed store's read of up_0; it reads `output` and writes the frame with the option off too
    total = down + up + store_extra
    return dict(pyramid_bytes=down + up, store_extra_bytes=store_extra, total_bytes=total, floor_us_at_3_35_TBps=round(total / HBM_BYTES_PER_S * 1e6, 2),
                pyramid_floor_us=round((down + up) / HBM_BYTES_PER_S * 1e6, 2))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--size", default="1920x1080")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    w, h = (int(v) for v in a.size.split("x"))
    res = dict(gpu=gpu_info(), size=f"{w}x{h}", rounds=a.rounds, frames_per_round=a.frames, bytes_model=bytes_model(w, h), scenes={})
    for name in ("cornell", "dungeon", "env_sunlit"):
        res["scenes"][name] = measure(getattr(scenes, name)(w, h), a, w, h)
    res["kernels_env_sunlit"] = kernel_times(scenes.env_sunlit(w, h), w, h)
    print(json.dumps(res, indent=1))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
