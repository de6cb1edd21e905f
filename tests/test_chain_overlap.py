"""A single-GPU Image-mode frame runs its ReSTIR DI chain on a second stream beside the GI chain (DESIGN.md §4 "Chain overlap").  The two
chains write disjoint buffers, so the overlapped frame must leave every buffer with the bits of the serial launch order: checked here
frame by frame against an engine held to the serial order, over 13 frames (every GI frame class: sampling, odd tracing / spatial, and
validation frames f % 6 >= 4), in the product default and the strict tier, on a caller's stream too."""
import ctypes as C

import numpy as np
import pytest

from strolle_b200 import scenes
from strolle_b200.engine import FORMAT_RGBA8_SRGB
from tests.util import CAMERA_BUFFERS, assert_bits_equal

FRAMES = 13
W, H = 200, 120


def _debug_serial_chains(e, serial):
    """st_debug_serial_chains (a development hook the public header leaves out): sets the engine's schedule, returns the number of
    frames it has rendered with the DI chain on its own stream."""
    fn = e.lib.st_debug_serial_chains
    fn.argtypes, fn.restype = [C.c_void_p, C.c_int, C.POINTER(C.c_uint64)], C.c_int
    n = C.c_uint64(0)
    e._check(fn(e._h, int(serial), C.byref(n)))
    return n.value


def _engine(blue_noise, exact, serial, scene):
    import strolle_b200
    e = strolle_b200.Engine(blue_noise=blue_noise, exact=exact)
    _debug_serial_chains(e, serial)
    return e, scenes.apply(e, scene)


def _scene(name):
    return getattr(scenes, name)(W, H)


def _compare(a, ca, b, cb, what):
    for name in CAMERA_BUFFERS:
        assert_bits_equal(a.read_buffer(ca, name), b.read_buffer(cb, name), f"{what}: {name}")


def _frames(pairs, frames=FRAMES):
    """Renders `frames` frames on every (engine, camera) pair, each delivering its Rgba8 frame, and checks every pair against the
    first (the serial engine) after each frame: all camera buffers and the Rgba8 bytes.  Returns the GI frame classes rendered."""
    ref_e, ref_c = pairs[0]
    hosts = [np.zeros((H, W, 4), np.uint8) for _ in pairs]
    seen = set()
    for _ in range(frames):
        f = ref_e.frame()
        seen.add("validation" if f % 6 >= 4 else "sampling" if f % 2 == 0 else "spatial")
        for (e, c), host in zip(pairs, hosts):
            e.tick(); e.render_camera(c, host, FORMAT_RGBA8_SRGB)
        for k, (e, c) in enumerate(pairs[1:], 1):
            _compare(ref_e, ref_c, e, c, f"engine {k}, frame {f}")
            assert np.array_equal(hosts[0], hosts[k]), f"engine {k}, frame {f}: Rgba8 frame differs"
    return seen


@pytest.mark.gpu
@pytest.mark.parametrize("exact", [False, True], ids=["product", "strict"])
@pytest.mark.parametrize("name", ["cornell", "dungeon"])
def test_overlapped_frame_is_the_serial_frame(blue_noise, name, exact):
    sc = _scene(name)
    serial = _engine(blue_noise, exact, True, sc)
    overlapped = _engine(blue_noise, exact, False, sc)
    assert _frames([serial, overlapped]) == {"validation", "sampling", "spatial"}
    assert _debug_serial_chains(serial[0], True) == 0
    assert _debug_serial_chains(overlapped[0], False) == FRAMES


@pytest.mark.gpu
def test_overlap_on_a_callers_stream(blue_noise):
    """The fork and the join are events on whatever stream the engine runs on: a torch stream, and the legacy default stream."""
    import torch
    sc = _scene("cornell")
    serial = _engine(blue_noise, False, True, sc)
    on_torch = _engine(blue_noise, False, False, sc)
    on_legacy = _engine(blue_noise, False, False, sc)
    stream = torch.cuda.Stream()
    on_torch[0].set_stream(stream.cuda_stream)
    on_legacy[0].set_stream(None)
    _frames([serial, on_torch, on_legacy], frames=8)
    for e, _ in (on_torch, on_legacy):
        assert _debug_serial_chains(e, False) == 8
    for e, _ in (serial, on_torch, on_legacy):
        e.close()


@pytest.mark.gpu
def test_serial_where_the_order_is_observed(blue_noise):
    """Timing mode (per-pass events), modes with one chain, and Reference mode keep the launch order; their frames are still the
    serial engine's."""
    for mode in (scenes.MODE_DI_DIFFUSE, scenes.MODE_GI_DIFFUSE, scenes.MODE_REFERENCE):
        sc = scenes.cornell(W, H, mode=mode)
        serial, plain = _engine(blue_noise, False, True, sc), _engine(blue_noise, False, False, sc)
        _frames([serial, plain], frames=6)
        assert _debug_serial_chains(plain[0], False) == 0, f"mode {mode} forked"
    sc = _scene("cornell")
    serial, timed = _engine(blue_noise, False, True, sc), _engine(blue_noise, False, False, sc)
    timed[0].enable_timing(True)
    _frames([serial, timed], frames=6)
    assert _debug_serial_chains(timed[0], False) == 0
    timed[0].enable_timing(False)
    _frames([serial, timed], frames=2)
    assert _debug_serial_chains(timed[0], False) == 2
