"""Chooses the shape of the bloom pyramid's small levels (ST_OPT_BLOOM) by measurement: builds the library once per variant (tuning
builds strolle_b200/_lib/libstrolle_b200_bloom_<name>.so with the ST_BLOOM_* macros of kernels.cu), then in a child process per variant
times the pyramid on scenes.cornell and scenes.env_sunlit at 1920x1080, product defaults (bloom defaults, L = 7).  Per variant and scene:
the device time per frame of the pyramid kernels (k_bloom_*) and their launches from torch.profiler, the median P_COMPOSITION slot
(the composition and the pyramid, launch gaps included; frames rendered without a copy) from the engine's pass timing, and whether the "bloom" words after
12 frames equal the default build's.  Prints the GPU's name and power limit and one JSON document.

Variants: `default` (one launch per level, down and up); the levels of at most 4096 texels (60x33 and smaller at 1080p, levels 4-6)
down and back up in one launch: `tail4k` (one CTA, passes over global memory), `smem4k` (one CTA holding the tail in its shared memory),
`cluster4k` (a cluster of 8 CTAs holding it in distributed shared memory); `cluster16k` (the cluster from 16384 texels, 120x67 at
1080p, levels 3-6).

    python tools/bloom_variants.py [--build-only] [--json out.json]
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
    "tail4k": ["ST_BLOOM_TAIL_TEXELS=4096"],
    "smem4k": ["ST_BLOOM_TAIL_TEXELS=4096", "ST_BLOOM_TAIL_KIND=1"],
    "cluster4k": ["ST_BLOOM_TAIL_TEXELS=4096", "ST_BLOOM_TAIL_KIND=2"],
    "cluster16k": ["ST_BLOOM_TAIL_TEXELS=16384", "ST_BLOOM_TAIL_KIND=2"],
}

CHILD = r"""
import hashlib, json, sys
import numpy as np, torch
from torch.profiler import ProfilerActivity, profile
import strolle_b200
from strolle_b200 import scenes
from strolle_b200.engine import FORMAT_RGBA8_SRGB, OPT_BLOOM
w, h = 1920, 1080
res = {}
for name in ("cornell", "env_sunlit"):
    e = strolle_b200.Engine()
    e.set_option(OPT_BLOOM, 1)
    cam = scenes.apply(e, getattr(scenes, name)(w, h))
    host = torch.zeros((h, w, 4), dtype=torch.uint8, pin_memory=True).numpy()
    for _ in range(12):
        e.tick(); e.render_camera(cam, host, FORMAT_RGBA8_SRGB)
    words = e.read_buffer(cam, "bloom").view(np.uint32)
    e.synchronize()
    frames = 24
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(frames):
            e.tick(); e.render_camera(cam, host, FORMAT_RGBA8_SRGB)
        e.synchronize()
    us = [ev.device_time_total for ev in prof.events() if ev.device_type.name == "CUDA" and "k_bloom_" in ev.name]
    # the P_COMPOSITION slot (device events around the composition, the pyramid and nothing else): launch gaps included
    slot = list(strolle_b200.PASS_NAMES).index("frame_composition")
    e.enable_timing(True); e.pass_times(reset=True)
    comp = []
    for _ in range(48):
        e.tick(); e.render_camera(cam)
        ms, _ = e.pass_times(reset=True)
        comp.append(float(ms[slot]) * 1e3)
    e.enable_timing(False)
    res[name] = dict(pyramid_us_per_frame=round(float(np.sum(us)) / frames, 2), launches_per_frame=len(us) / frames,
                     composition_slot_us_p50=round(float(np.median(comp)), 1), words_sha1=hashlib.sha1(words.tobytes()).hexdigest())
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
    libs = {name: build.build(defines=d, tag="bloom_" + name) for name, d in VARIANTS.items()}
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
        out["variants"][name] = {s: dict(pyramid_us_per_frame=r["pyramid_us_per_frame"], launches_per_frame=r["launches_per_frame"],
                                         composition_slot_us_p50=r["composition_slot_us_p50"],
                                         same_words_as_default=(s in ref and r["words_sha1"] == ref[s]["words_sha1"]))
                                 for s, r in v.items()}
    print(json.dumps(out, indent=1))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
