"""What running the ReSTIR DI chain on a second stream beside the GI chain (DESIGN.md §4 "Chain overlap") buys on the GPU:
scenes.cornell and scenes.dungeon at 1920x1080, product-tier defaults.  One engine per scene renders blocks of --frames frames (two
GI cycles by default) with the serial and the overlapped schedule alternated over --rounds rounds, switched through the development
hook st_debug_serial_chains.  Each block is timed like bench.py's main line: CUDA events on the engine stream around back-to-back
st_tick + st_render_camera calls.  Prints the GPU's name, power limit and SM clock, and per scene the median ms per frame of each
schedule with its p10-p90 spread over the blocks, the gain, and (from a timed serial run) the per-pass table and each chain's share.

    python tools/chain_overlap_cost.py [--rounds 10] [--frames 12] [--size 1920x1080] [--json out.json]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import strolle_b200
from strolle_b200 import scenes


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def serial_chains(e, serial):
    fn = e.lib.st_debug_serial_chains
    fn.argtypes, fn.restype = [C.c_void_p, C.c_int, C.POINTER(C.c_uint64)], C.c_int
    n = C.c_uint64(0)
    e._check(fn(e._h, int(serial), C.byref(n)))
    return n.value


def block_ms(e, cam, frames):
    e.mark_begin()
    for _ in range(frames):
        e.tick(); e.render_camera(cam)
    return e.mark_end() / frames


def pass_table(e, cam, frames):
    """Per-pass device ms per frame of the serial schedule (timing mode always runs it), and the DI / GI chains' sums."""
    e.enable_timing(True); e.pass_times(reset=True)
    for _ in range(frames):
        e.tick(); e.render_camera(cam)
    ms, launches = e.pass_times(reset=True)
    e.enable_timing(False)
    names = list(strolle_b200.PASS_NAMES)
    table = {names[i]: round(float(ms[i]) / frames, 4) for i in range(len(names)) if launches[i]}
    di = sum(v for k, v in table.items() if k.startswith("di_"))
    gi = sum(v for k, v in table.items() if k.startswith("gi_"))
    return table, dict(di_chain_ms=round(di, 4), gi_chain_ms=round(gi, 4), all_passes_ms=round(sum(table.values()), 4))


def measure(scene, a):
    e = strolle_b200.Engine()
    cam = scenes.apply(e, scene)
    for serial in (True, False):   # warm both schedules over every GI frame class
        serial_chains(e, serial)
        block_ms(e, cam, a.frames)
    times = {"serial": [], "overlapped": []}
    for r in range(a.rounds):
        for serial in ((True, False) if r % 2 == 0 else (False, True)):
            serial_chains(e, serial)
            times["serial" if serial else "overlapped"].append(block_ms(e, cam, a.frames))
    overlapped_frames = serial_chains(e, False)
    q = lambda v: [round(float(np.percentile(v, p)), 4) for p in (50, 10, 90)]
    res = {k: dict(ms_per_frame_p50_p10_p90=q(v)) for k, v in times.items()}
    s, o = float(np.median(times["serial"])), float(np.median(times["overlapped"]))
    res["gain_ms"] = round(s - o, 4)
    res["gain_pct"] = round(100.0 * (s - o) / s, 2)
    res["overlapped_frames"] = overlapped_frames
    res["pass_ms_per_frame"], res["chains"] = pass_table(e, cam, a.frames)
    e.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--frames", type=int, default=12)
    ap.add_argument("--size", default="1920x1080")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    w, h = (int(v) for v in a.size.split("x"))
    res = dict(gpu=gpu_info(), size=f"{w}x{h}", rounds=a.rounds, frames_per_block=a.frames, scenes={})
    for name in ("cornell", "dungeon"):
        res["scenes"][name] = measure(getattr(scenes, name)(w, h), a)
    print(json.dumps(res, indent=1))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
