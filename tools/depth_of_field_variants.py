"""Chooses how the depth-of-field gather (ST_OPT_DEPTH_OF_FIELD) reads its taps by measurement: builds the library once per variant
(the default library, and tuning builds strolle_b200/_lib/libstrolle_b200_dof_<name>.so with the ST_DOF_STAGE_MAX_RADIUS macro of
kernels.cu), then in a child process per
variant times k_dof_gather on scenes.cornell and scenes.env_sunlit at 1920x1080 at max_radius 16 and 32 (the heavy lens of
tools/depth_of_field_cost.py) and checks that the "depth_of_field" words and the Rgba32F frame after 12 frames equal the default build's.
Prints the GPU's name and power limit and one JSON document.

Variants: `stage` (each gathering tile's colours and radii, with a halo of its radius, staged in shared memory), `global` (every tap
read from global memory, through L1 / L2) and `default` (the stage up to max_radius 16, global memory above).

    python tools/depth_of_field_variants.py [--build-only] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

VARIANTS = {"default": [], "global": ["ST_DOF_STAGE_MAX_RADIUS=0"], "stage": ["ST_DOF_STAGE_MAX_RADIUS=32"]}

CHILD = r"""
import hashlib, json
import numpy as np
from torch.profiler import ProfilerActivity, profile
from strolle_b200 import scenes
from strolle_b200.engine import FORMAT_RGBA32F
from tools.depth_of_field_cost import engine
res = {}
for name in ("cornell", "env_sunlit"):
    for R in (16, 32):
        sc = getattr(scenes, name)(1920, 1080)
        e, cam, host = engine(sc, R)
        words = e.read_buffer(cam, "depth_of_field").view(np.uint32)
        e.copy_output(cam, host, FORMAT_RGBA32F)
        digest = hashlib.sha1(words.tobytes() + host.view(np.uint32).tobytes()).hexdigest()
        frames = 16
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(frames):
                e.tick(); e.render_camera(cam, host, FORMAT_RGBA32F)
            e.synchronize()
        us = [ev.device_time_total for ev in prof.events() if ev.device_type.name == "CUDA" and "k_dof_gather" in ev.name]
        res[f"{name}_R{R}"] = dict(gather_us_median=round(float(np.median(us)), 2), sha1=digest)
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
    libs = {name: build.build(defines=d, tag="dof_" + name) if d else build.build() for name, d in VARIANTS.items()}
    if a.build_only:
        print(json.dumps(libs, indent=1))
        return
    table = {}
    for name, lib in libs.items():
        r = subprocess.run([sys.executable, "-c", CHILD], env=dict(os.environ, STROLLE_B200_LIB=lib), cwd=ROOT, capture_output=True, text=True)
        line = [l for l in r.stdout.splitlines() if l.startswith("RESULT ")]
        table[name] = json.loads(line[0][7:]) if (line and not r.returncode) else dict(error=(r.stdout + r.stderr)[-600:])
    ref = table.get("default", {})
    out = dict(gpu=gpu_info(), size="1920x1080", variants={})
    for name, v in table.items():
        out["variants"][name] = v if "error" in v else {
            k: dict(gather_us_median=x["gather_us_median"], same_words_and_frame_as_default=(k in ref and x["sha1"] == ref[k]["sha1"]))
            for k, x in v.items()}
    print(json.dumps(out, indent=1))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
