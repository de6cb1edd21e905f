#!/usr/bin/env python
"""Run under torchrun on N GPUs: the tonemapped Rgba8 store with a fixed exposure (ST_OPT_TONEMAPPING = 4, AgX) on row strips, through
both gathers of st_render_strips (1: strips assembled on rank 0; 2: every rank copies its own rows into one shared host frame, here
compared row by row on each rank), is the single-GPU frame bit for bit; with ST_OPT_AUTO_EXPOSURE on, st_render_strips is refused.
Prints one OK/FAIL line per check on rank 0.

    python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 tools/verify_multigpu_exposure.py
"""
import os
import sys

os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import torch.distributed as dist

import strolle_b200
from strolle_b200 import scenes
from strolle_b200.engine import FORMAT_RGBA8_SRGB, OPT_AUTO_EXPOSURE, OPT_TONEMAPPING
from strolle_b200.multigpu import StripRunner, strip_bounds

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
W, H, FRAMES = 640, 360 * world, 5
scene = scenes.cornell(W, H)


def tonemapped(e):
    e.set_option(OPT_TONEMAPPING, 4)
    e.set_exposure(ev=-0.75, compensation=0.25)
    return e


def check(gather):
    eng = tonemapped(strolle_b200.Engine(device=local))
    cam = scenes.apply(eng, scene)
    runner = StripRunner(eng, cam, W, H, rank, world, native=True, peer=True)
    full = tonemapped(strolle_b200.Engine(device=local))
    cfull = scenes.apply(full, scene)
    y0, y1 = strip_bounds(H, world)[rank]
    ok = True
    for f in range(FRAMES):
        got, want = np.zeros((H, W, 4), np.uint8), np.zeros((H, W, 4), np.uint8)
        eng.tick(); full.tick()
        runner.render(out=got, fmt=FORMAT_RGBA8_SRGB, gather=gather)
        eng.synchronize()
        full.render_camera(cfull, want, FORMAT_RGBA8_SRGB)
        same = (got == want) if gather == 1 else (got[y0:y1] == want[y0:y1])
        if (gather == 2 or rank == 0) and not same.all():
            ok = False
            print(f"FAIL rank {rank} gather {gather} frame {f + 1}: {int((~same).sum())} bytes differ", flush=True)
    flag = torch.tensor([int(ok)], device="cuda")
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    if rank == 0:
        print(f"{'OK' if flag.item() else 'FAIL'} tonemapped strips (AgX, fixed exposure), gather {gather}: {world} ranks x {W}x{H // world} rows, "
              f"{FRAMES} frames bit-identical to the single GPU", flush=True)
    eng.set_option(OPT_AUTO_EXPOSURE, 1); eng.tick()
    try:
        eng.render_strips(cam, None, FORMAT_RGBA8_SRGB)
        refused = False
    except strolle_b200.StrolleError:
        refused = True
    if rank == 0:
        print(f"{'OK' if refused else 'FAIL'} auto exposure refused on strips", flush=True)
    dist.barrier()


check(1)
check(2)
dist.destroy_process_group()
