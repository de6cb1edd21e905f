"""Chooses the shape of the exposure histogram (k_exposure_histogram, ST_OPT_AUTO_EXPOSURE) by measurement: builds the library once per
variant (tuning builds strolle_b200/_lib/libstrolle_b200_expo_<name>.so with the ST_EXPO_* macros of kernels.cu), then in a child
process per variant times the metering on scenes.cornell and scenes.env_sunlit (a sky: whole warps in one bin) at 1920x1080, product
defaults, AgX + auto exposure.  Per variant and scene: the median device time per frame of the metering kernels (k_exposure_histogram,
plus k_exposure_meter where the metering is a second launch) from torch.profiler, and whether the exposure words after 12 frames equal
the default build's.  Prints the GPU's name and power limit and one JSON document.

Variants: `default` (512 threads, 4 CTAs per SM, lanes merged per bin with __match_any_sync, metering in the last CTA); `no_match`
(a shared atomicAdd per lane instead); `second_launch` (the metering in its own one-CTA launch); `cta1` / `cta2` (1 or 2 CTAs per SM);
`t256` (256 threads, 8 CTAs per SM).

    python tools/exposure_variants.py [--build-only] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

VARIANTS = {
    "default": [],
    "no_match": ["ST_EXPO_AGGREGATE=0"],
    "second_launch": ["ST_EXPO_METER_LAUNCH=1"],
    "cta1": ["ST_EXPO_CTAS_PER_SM=1"],
    "cta2": ["ST_EXPO_CTAS_PER_SM=2"],
    "t256": ["ST_EXPO_THREADS=256", "ST_EXPO_CTAS_PER_SM=8"],
}

CHILD = r"""
import json, sys
import numpy as np, torch
from torch.profiler import ProfilerActivity, profile
import strolle_b200
from strolle_b200 import scenes
from strolle_b200.engine import FORMAT_RGBA8_SRGB, OPT_AUTO_EXPOSURE, OPT_TONEMAPPING, TONEMAP_AGX
w, h = 1920, 1080
res = {}
for name in ("cornell", "env_sunlit"):
    e = strolle_b200.Engine()
    e.set_option(OPT_TONEMAPPING, TONEMAP_AGX); e.set_option(OPT_AUTO_EXPOSURE, 1)
    cam = scenes.apply(e, getattr(scenes, name)(w, h))
    host = torch.zeros((h, w, 4), dtype=torch.uint8, pin_memory=True).numpy()
    for _ in range(12):
        e.tick(); e.render_camera(cam, host, FORMAT_RGBA8_SRGB)
    words = e.read_buffer(cam, "exposure").view(np.uint32)
    e.synchronize()
    frames = 24
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(frames):
            e.tick(); e.render_camera(cam, host, FORMAT_RGBA8_SRGB)
        e.synchronize()
    us = [ev.device_time_total for ev in prof.events() if ev.device_type.name == "CUDA" and "k_exposure_" in ev.name]
    res[name] = dict(metering_us_per_frame=round(float(np.sum(us)) / frames, 2), launches=len(us), words=words.tolist())
print("RESULT " + json.dumps(res))
"""


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--build-only", action="store_true")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    from strolle_b200 import build
    libs = {name: build.build(defines=d, tag="expo_" + name) for name, d in VARIANTS.items()}
    if a.build_only:
        print(json.dumps(libs, indent=1))
        return
    table = {}
    for name, lib in libs.items():
        r = subprocess.run([sys.executable, "-c", CHILD], env=dict(os.environ, STROLLE_B200_LIB=lib), cwd=ROOT, capture_output=True, text=True)
        line = [l for l in r.stdout.splitlines() if l.startswith("RESULT ")]
        if r.returncode or not line:
            table[name] = dict(error=(r.stdout + r.stderr)[-600:])
            continue
        table[name] = json.loads(line[0][7:])
    ref = table.get("default", {})
    out = dict(gpu=gpu_info(), size="1920x1080", variants={})
    for name, v in table.items():
        if "error" in v:
            out["variants"][name] = v
            continue
        out["variants"][name] = {s: dict(metering_us_per_frame=r["metering_us_per_frame"], launches=r["launches"],
                                         same_words_as_default=(s in ref and r["words"] == ref[s]["words"])) for s, r in v.items()}
    print(json.dumps(out, indent=1))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
