"""Temporal anti-aliasing (ST_OPT_TEMPORAL_AA): the oracle extension against the plain oracle with the option off and in the modes it
leaves alone, against the float64 restatement (with its deliberate mistakes), the purpose of the option on the oracle, and the CUDA
path against the extension (every camera buffer and both history buffers of the strict tier, the product tier's resolve on its own
inputs, the option's selection, the statistic, the strip entry points)."""
import math

import numpy as np
import pytest

from strolle_b200 import scenes
from oracle import pyoracle
from oracle_taa import pyoracle_taa as T
from tests import ref64_taa as R
from tests.util import CAMERA_BUFFERS, assert_bits_equal, rel_l2

OPT_TEMPORAL_AA, STAT_TAA_RESOLVES = 18, 12
OPT_NORMAL_MAPS, OPT_TEXTURE_FILTER, OPT_LIGHT_GRID = 14, 17, 16
HISTORY = ("taa_history_a", "taa_history_b")


def _taa_oracle(blue_noise, scene, on=True, mutation=None):
    eo = T.TemporalAAOracleEngine(blue_noise=blue_noise, mutation=mutation)
    eo.set_temporal_aa(on)
    return eo, scenes.apply(eo, scene)


MOVING = {"aa_edges": 321, "cornell": 305, "textured_room": 304, "dungeon_synthetic": None, "tiled_ground": 313, "normal_mapped_room": None}


def _pose(scene, f):
    c = scene["camera"]
    t = np.asarray(c["transform"], np.float32).reshape(4, 4).copy()
    t[3, :3] += np.array([0.02 * f, -0.01 * f, -0.03 * f], np.float32)
    return t.reshape(-1)


def _step(engines, scene, f, w, h, render=True):
    """Frame f: the camera drifts; one instance (where the scene has a listed one) moves too."""
    c = scene["camera"]
    inst = MOVING.get(scene["name"])
    for e, cam in engines:
        e.update_camera(cam, c["mode"], c["denoise"], c["ref_depth"], w, h, _pose(scene, f), c["projection"])
        if inst is not None:
            _, mesh, mat, _ = next(i for i in scene["instances"] if i[0] == inst)
            e.insert_instance(inst, mesh, mat, np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0.03 * f, 0.0, 0.02 * f], np.float32))
        e.tick()
        if render:
            e.render_camera(cam)


# ---- CPU ------------------------------------------------------------------------------------------------------------------------

def test_jitter_sequence():
    """J(f) is the 16-entry Halton (2, 3) sequence minus 0.5, J(0) = J(16), and the extension's float32 values are the rule's."""
    for f in range(0, 40):
        assert np.allclose(T.jitter(f), R.jitter(f), atol=2.0 ** -24), f
    assert (T.jitter(0) == T.jitter(16)).all() and (T.jitter(17) == T.jitter(1)).all()
    assert np.allclose(T.jitter(1), (0.0, -1.0 / 6.0)) and np.allclose(T.jitter(2), (-0.25, 1.0 / 6.0))
    js = np.stack([T.jitter(f) for f in range(1, 17)])
    assert len({tuple(j) for j in js}) == 16 and (np.abs(js) < 0.5).all()


@pytest.mark.parametrize("mode", [scenes.MODE_IMAGE, scenes.MODE_GI_DIFFUSE])
def test_oracle_option_off_is_the_oracle(blue_noise, mode):
    """With the option off the extension is the plain oracle, bit for bit, in every camera buffer over 5 moving frames."""
    w, h = 64, 48
    sc = scenes.cornell(w, h, mode=mode)
    off, coff = _taa_oracle(blue_noise, sc, on=False)
    plain = pyoracle.OracleEngine(blue_noise=blue_noise)
    cp = scenes.apply(plain, sc)
    for f in range(5):
        _step([(off, coff), (plain, cp)], sc, f, w, h)
        for n in CAMERA_BUFFERS + ["curr_camera", "prev_camera"]:
            assert_bits_equal(off.read_buffer(coff, n), plain.read_buffer(cp, n), f"frame {f + 1} {n}")


@pytest.mark.parametrize("mode", [scenes.MODE_REFERENCE, scenes.MODE_BVH_HEATMAP])
def test_oracle_reference_and_heatmap_untouched(blue_noise, mode):
    """Reference mode and the heat map are neither jittered nor resolved: option on equals option off, bit for bit."""
    w, h = 64, 48
    sc = scenes.cornell(w, h, mode=mode)
    on, con = _taa_oracle(blue_noise, sc)
    off, coff = _taa_oracle(blue_noise, sc, on=False)
    for f in range(4):
        _step([(on, con), (off, coff)], sc, f, w, h)
        for n in CAMERA_BUFFERS + ["curr_camera", "prev_camera"]:
            assert_bits_equal(on.read_buffer(con, n), off.read_buffer(coff, n), f"frame {f + 1} {n}")


def _float64_frames(blue_noise, name, mutation=None, frames=13, w=64, h=40):
    sc = scenes.aa_edges(w, h) if name == "aa_edges" else getattr(scenes, name)(w, h)
    eo, cam = _taa_oracle(blue_noise, sc, mutation=mutation)
    eo.probe = True
    c = sc["camera"]
    stats = []
    for f in range(frames):
        prev_t = _pose(sc, f - 1) if f else np.asarray(c["transform"], np.float32)
        _step([(eo, cam)], sc, f, w, h, render=False)
        fid = int(eo.lib.orc_frame(eo.h)) - 1
        cur = 1 if fid % 2 == 1 else 0
        hist_in = eo.history(cam)[cur ^ 1].copy()   # last frame's slot: a when this frame writes b
        eo.render_camera(cam)
        R.check_camera(_pose(sc, f), c["projection"], w, h, fid, eo.read_buffer(cam, "curr_camera"))
        R.check_camera(prev_t, c["projection"], w, h, fid - 1, eo.read_buffer(cam, "prev_camera"))
        d0 = eo.read_buffer(cam, "prim_gbuffer_d0_" + "ab"[cur]).reshape(-1, 4)[:, 0]
        stats.append(R.check_resolve(w, h, fid, eo.last_probe, d0, eo.read_buffer(cam, "velocity_map"), eo.read_buffer(cam, "curr_camera"),
                                     eo.read_buffer(cam, "prev_camera"), hist_in, eo.history(cam)[cur], eo.read_buffer(cam, "output")))
    return stats


@pytest.mark.parametrize("name", ["aa_edges", "cornell", "textured_room"])
def test_oracle_inside_float64_bound(blue_noise, name):
    """13 frames with the camera and an instance moving: the jittered cameras and every stage of the resolve lie inside the float64
    bound; undecided choices are counted."""
    stats = _float64_frames(blue_noise, name)
    worst = max(s["worst"] for s in stats)
    und = {k: sum(s[k] for s in stats) for k in ("undecided_onscreen", "undecided_floor", "undecided_clip")}
    print(f"{name}: worst error / bound {worst:.3g}, undecided {und}")
    assert worst <= 1.0


@pytest.mark.parametrize("mutation", sorted(T.MUTATIONS))
def test_oracle_mutation_leaves_float64_bound(blue_noise, mutation):
    """Each deliberate mistake of the extension makes the float64 check fail (textured_room shows sky to the sky-point mistake)."""
    with pytest.raises(AssertionError):
        _float64_frames(blue_noise, "textured_room", mutation=mutation, frames=6)


AA_W, AA_H, AA_S = 96, 64, 8


def _aa_frames(blue_noise, on, frames, pan, w=AA_W, h=AA_H, first=0):
    """aa_edges with the camera panning `pan` pixels per frame (at the depth of the emissive shapes); the resolved (or composed) frames."""
    sc = scenes.aa_edges(w, h)
    e, cam = _taa_oracle(blue_noise, sc, on=on)
    c = sc["camera"]
    px = 2.0 * 4.9 * math.tan(math.pi / 8.0) / (h // (AA_S if w > AA_W else 1))
    out = []
    for f in range(first, first + frames):
        t = np.asarray(c["transform"], np.float32).reshape(4, 4).copy()
        t[3, 0] += np.float32(pan * (f - 16) * px)
        e.update_camera(cam, c["mode"], c["denoise"], c["ref_depth"], w, h, t.reshape(-1), c["projection"])
        e.tick(); e.render_camera(cam)
        out.append(e.read_buffer(cam, "output").reshape(h, w, 4)[..., :3].astype(np.float64))
    return out, e, cam


def _aa_error(blue_noise, pan, on_frames):
    big = _aa_frames(blue_noise, False, 1, pan, AA_W * AA_S, AA_H * AA_S, first=31)[0][0]
    blk = big.reshape(AA_H, AA_S, AA_W, AA_S, 3)
    truth, edge = blk.mean((1, 3)), (blk.max((1, 3)) != blk.min((1, 3))).any(-1)
    err = lambda a: float(np.abs(a - truth)[edge].mean())
    return err(on_frames[-1]), err(_aa_frames(blue_noise, False, 32, pan)[0][-1]), int(edge.sum())


def test_antialiasing_static_and_panning(blue_noise):
    """The purpose, on the oracle: after 32 frames of aa_edges, the mean absolute error of the edge pixels (8x8 blocks of an 8x8-
    supersampled option-off render that are not uniform) against that render, box-averaged, is at most half the option-off error (static
    camera; measured 0.368), and with the camera panning 1 pixel per frame at most 1.5 times the static ratio."""
    on, _, _ = _aa_frames(blue_noise, True, 32, 0)
    e_on, e_off, n = _aa_error(blue_noise, 0, on)
    static = e_on / e_off
    pan_on, _, _ = _aa_frames(blue_noise, True, 32, 1)
    p_on, p_off, pn = _aa_error(blue_noise, 1, pan_on)
    print(f"aa_edges: static ratio {static:.3f} ({n} edge pixels), panning ratio {p_on / p_off:.3f} ({pn} edge pixels)")
    assert n > 100 and pn > 100
    assert static <= 0.5
    assert p_on / p_off <= 1.5 * static


def test_constant_neighbourhood_and_offscreen(blue_noise):
    """Camera and the quad moving on aa_edges (a noise-free frame): wherever the 3x3 composed neighbourhood is constant the resolved pixel equals it
    within 1e-6 relative (plus what the clip's 1e-8 epsilon on the box extent allows around a black constant), and pixels whose history position falls off screen store a count of 1 (n = 0 plus this frame) and output
    the composed colour (within the tonemap round trip)."""
    w, h = 64, 40
    sc = scenes.aa_edges(w, h)
    eo, cam = _taa_oracle(blue_noise, sc)
    eo.probe = True
    seen_const = seen_off = 0
    for f in range(13):
        _step([(eo, cam)], sc, -4 * f, w, h)   # the camera backs away: border pixels come from outside last frame
        pr = eo.last_probe.reshape(h, w, T.PROBE_WORDS)
        c = pr[..., 18:21].astype(np.float64)
        out = eo.read_buffer(cam, "output").reshape(h, w, 4)[..., :3].astype(np.float64)
        cp = np.pad(c, ((1, 1), (1, 1), (0, 0)), mode="edge")
        const = np.ones((h, w), bool)
        for dy in range(3):
            for dx in range(3):
                const &= (cp[dy:dy + h, dx:dx + w] == c).all(-1)
        # a clipped history lies within the box's epsilon (1e-8 per YCoCg component, 3e-8 per tonemapped channel) of the constant
        tol = 1e-6 * np.abs(c) + 3e-8 * (1.0 + c.max(-1, keepdims=True)) ** 2
        assert (np.abs(out - c)[const] <= tol[const]).all(), f"frame {f + 1}: {np.abs(out - c)[const].max()}"
        off = pr[..., 2] == 0
        hist = eo.history(cam)[1 if (int(eo.lib.orc_frame(eo.h)) - 1) % 2 == 1 else 0].reshape(h, w, 4)
        assert (hist[..., 3][off] == 1.0).all()
        assert (np.abs(out - c)[off] <= 1e-6 * np.abs(c)[off] + 1e-30).all()
        seen_const += int(const.sum()); seen_off += int(off.sum())
    assert seen_const > 1000 and seen_off > 50, (seen_const, seen_off)


def test_option_constants_agree():
    """The header, the Python package and the Rust sys crate agree on the option and the statistic."""
    import os
    import re
    from strolle_b200 import engine
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    hdr = open(os.path.join(root, "include", "strolle_b200.h")).read()
    rs = open(os.path.join(root, "rust", "strolle-b200-sys", "src", "lib.rs")).read()
    for name, value, py in (("ST_OPT_TEMPORAL_AA", 18, engine.OPT_TEMPORAL_AA), ("ST_STAT_TAA_RESOLVES", 12, engine.STAT_TAA_RESOLVES)):
        assert re.search(rf"\b{name} = {value}\b", hdr), name
        assert re.search(rf"\b{name}: c_int = {value};", rs), name
        assert py == value, name


# ---- GPU ------------------------------------------------------------------------------------------------------------------------

def _gpu_engine(blue_noise, exact, taa=True, fused=None):
    import strolle_b200
    e = strolle_b200.Engine(blue_noise=blue_noise, exact=exact)
    e.set_option(OPT_TEMPORAL_AA, int(taa))
    if fused is not None:
        from strolle_b200.engine import OPT_FUSED_PASSES
        e.set_option(OPT_FUSED_PASSES, int(fused))
    return e


def _scene(name, w, h, **kw):
    return scenes.aa_edges(w, h, **kw) if name == "aa_edges" else getattr(scenes, name)(w, h, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("name,mode,denoise", [("cornell", scenes.MODE_IMAGE, True), ("cornell", scenes.MODE_IMAGE, False),
                                               ("textured_room", scenes.MODE_IMAGE, True), ("aa_edges", scenes.MODE_IMAGE, True),
                                               ("cornell", scenes.MODE_DI_DIFFUSE, True), ("cornell", scenes.MODE_GI_SPECULAR, False)])
@pytest.mark.parametrize("size", [(224, 126), (67, 45)])
@pytest.mark.parametrize("fused", [False, True])
def test_strict_tier_bit_exact_with_oracle(oracle, blue_noise, name, mode, denoise, size, fused):
    """Option on, strict arithmetic, 13 frames with the camera and an instance moving: every camera buffer, both history buffers and the
    jittered cameras are the extension's, bit for bit (the fused schedule: every buffer it still writes)."""
    from tests.test_gpu_parity import NOT_WRITTEN_WHEN_FUSED
    w, h = size
    scene = _scene(name, w, h, mode=mode, denoise=denoise)
    eg = _gpu_engine(blue_noise, True, fused=fused)
    cg = scenes.apply(eg, scene)
    eo, co = _taa_oracle(blue_noise, scene)
    # without the denoiser the fused DI spatial launch's scratch (K8's colours and stash) is left unwritten and nothing reads it
    skip = (NOT_WRITTEN_WHEN_FUSED | ({"di_diff_curr_colors", "di_diff_stash", "gi_diff_curr_colors", "gi_diff_stash"} if not denoise else set())) if fused else set()
    names = [n for n in CAMERA_BUFFERS if n not in skip] + list(HISTORY) + ["curr_camera", "prev_camera"]
    for f in range(13):
        _step([(eg, cg), (eo, co)], scene, f, w, h)
        for n in names:
            assert_bits_equal(eg.read_buffer(cg, n), eo.read_buffer(co, n), f"{name} mode {mode} fused={fused} {size} frame {f + 1} {n}")


@pytest.mark.gpu
def test_strict_tier_with_other_options(oracle, blue_noise):
    """Normal maps, the texture filter and the light grid on together with the option: the output and both history buffers are those
    of the option-on extension run on the option-on device buffers (the strict tier's resolve on its own inputs), over 13 frames."""
    w, h = 224, 126
    scene = scenes.normal_mapped_room(w, h)
    eg = _gpu_engine(blue_noise, True)
    for o, v in ((OPT_NORMAL_MAPS, 1), (OPT_TEXTURE_FILTER, 1), (OPT_LIGHT_GRID, 8)):
        eg.set_option(o, v)
    cg = scenes.apply(eg, scene)
    _resolve_matches_restatement(eg, cg, scene, w, h, frames=13)


def _resolve_matches_restatement(eg, cg, scene, w, h, frames):
    """Steps the device frame by frame; before each resolve, reads its inputs and checks the resolve's output and history against
    the extension's resolve over those inputs, bit for bit."""
    from tests.util import Frame
    c = scene["camera"]
    for f in range(frames):
        eg.update_camera(cg, c["mode"], c["denoise"], c["ref_depth"], w, h, _pose(scene, f), c["projection"])
        eg.tick()
        fr = Frame(eg, cg, w, h)
        k = fr.steps(T.P_COMPOSITION)[-1]
        fr.run_to(k - 1)
        fid = eg.frame() - 1
        cur = 1 if fid % 2 == 1 else 0
        den = c["denoise"]
        bufs = dict(d0=fr.read("prim_gbuffer_d0_" + "ab"[cur]), d1=fr.read("prim_gbuffer_d1_" + "ab"[cur]),
                    di_diff=fr.read("di_diff_curr_colors" if den else "di_diff_samples"), di_spec=fr.read("di_spec_samples"),
                    gi_diff=fr.read("gi_diff_curr_colors" if den else "gi_diff_samples"), gi_spec=fr.read("gi_spec_samples"),
                    ref_colors=fr.read("ref_colors"), vel=fr.read("velocity_map"))
        try:
            hist_in = eg.read_buffer(cg, HISTORY[cur ^ 1])
        except Exception:
            hist_in = np.zeros(w * h * 4, np.float32)
        jit = np.concatenate([T.jitter(fid), T.jitter(fid - 1)])
        want_h, want_o = T.resolve_arrays(w, h, c["mode"], cur, bufs, eg.read_buffer(cg, "curr_camera"), eg.read_buffer(cg, "prev_camera"), jit, hist_in)
        fr.run_to(k)
        assert_bits_equal(eg.read_buffer(cg, "output"), want_o, f"frame {f + 1} output")
        assert_bits_equal(eg.read_buffer(cg, HISTORY[cur]), want_h, f"frame {f + 1} history")


def _product_drift(blue_noise, scene, w, h, taa):
    """Worst relative per-channel L2 of the product tier's output against the oracle (the extension with the option as given) over
    13 moving frames."""
    prod = _gpu_engine(blue_noise, False, taa=taa)
    cp = scenes.apply(prod, scene)
    eo, co = _taa_oracle(blue_noise, scene, on=taa)
    worst = 0.0
    for f in range(13):
        _step([(prod, cp), (eo, co)], scene, f, w, h)
        a, b = prod.read_buffer(cp, "output").reshape(-1, 4)[:, :3], eo.read_buffer(co, "output").reshape(-1, 4)[:, :3]
        worst = max([worst] + [rel_l2(a[:, ch], b[:, ch]) for ch in range(3)])
    return worst


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["cornell", "dungeon"])
def test_product_tier(oracle, blue_noise, name):
    """Product defaults: given the device's own G-buffer, signals, velocity map and history, the resolve's output and history are the
    restatement's bit for bit (13 frames).  The resolved frame stays within 1e-3 relative per-channel L2 of the extension, or, where
    the fast-shading tier's own drift from the oracle is larger with the option off (the sunlit dungeon), within 1.5 times that drift:
    the resolve blends frames, it adds no error of its own."""
    w, h = 224, 126
    scene = _scene(name, w, h)
    prod = _gpu_engine(blue_noise, False)
    cp = scenes.apply(prod, scene)
    _resolve_matches_restatement(prod, cp, scene, w, h, frames=13)
    on, off = _product_drift(blue_noise, scene, w, h, True), _product_drift(blue_noise, scene, w, h, False)
    print(f"{name}: worst relative L2 option on {on:.3g}, option off {off:.3g}")
    assert on <= max(1e-3, 1.5 * off)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [scenes.MODE_REFERENCE, scenes.MODE_BVH_HEATMAP])
def test_reference_and_heatmap_untouched(blue_noise, mode):
    """Reference mode and the heat map with the option on are bit-identical to the option off; nothing is resolved."""
    w, h = 96, 64
    sc = scenes.cornell(w, h, mode=mode)
    on, off = _gpu_engine(blue_noise, False), _gpu_engine(blue_noise, False, taa=False)
    con, coff = scenes.apply(on, sc), scenes.apply(off, sc)
    for f in range(4):
        _step([(on, con), (off, coff)], sc, f, w, h)
        for n in CAMERA_BUFFERS + ["curr_camera", "prev_camera"]:
            assert_bits_equal(on.read_buffer(con, n), off.read_buffer(coff, n), f"frame {f + 1} {n}")
    assert on.get_stat(STAT_TAA_RESOLVES) == 0


@pytest.mark.gpu
def test_option_statistic_and_history_lifetime(blue_noise):
    """Values other than 0 and 1 are refused; ST_STAT_TAA_RESOLVES counts resolves; the history exists only while the option is on
    and restarts when it turns on again and when the camera is reallocated."""
    w, h = 64, 48
    sc = scenes.cornell(w, h)
    e = _gpu_engine(blue_noise, False)
    for bad in (-1, 2, 18):
        with pytest.raises(Exception):
            e.set_option(OPT_TEMPORAL_AA, bad)
    cam = scenes.apply(e, sc)
    for f in range(3):
        e.tick(); e.render_camera(cam)
    assert e.get_stat(STAT_TAA_RESOLVES) == 3
    assert e.read_buffer(cam, "taa_history_b").reshape(-1, 4)[:, 3].max() == 3.0   # frame 3 wrote b
    e.set_option(OPT_TEMPORAL_AA, 0); e.tick(); e.render_camera(cam)
    assert e.get_stat(STAT_TAA_RESOLVES) == 3
    with pytest.raises(Exception):
        e.read_buffer(cam, "taa_history_a")
    e.set_option(OPT_TEMPORAL_AA, 1); e.tick(); e.render_camera(cam)
    assert e.read_buffer(cam, "taa_history_b").reshape(-1, 4)[:, 3].max() == 1.0   # frame 5 wrote b from an empty history
    c = sc["camera"]
    e.update_camera(cam, c["mode"], False, c["ref_depth"], w, h, c["transform"], c["projection"])   # reallocation
    e.tick(); e.render_camera(cam)
    assert e.read_buffer(cam, "taa_history_a").reshape(-1, 4)[:, 3].max() == 1.0   # frame 6 restarted too
    assert e.get_stat(STAT_TAA_RESOLVES) == 5


@pytest.mark.gpu
def test_strips_refused_and_engine_usable(blue_noise):
    """With the option on, row strips (a two-member group on the one device) return ST_ERR_INVALID without enqueuing anything, and
    the group renders again once the option is off; a single engine keeps rendering with the option on."""
    import strolle_b200
    w, h = 256, 288
    sc = scenes.cornell(w, h)
    grp = strolle_b200.MultiEngine([0, 0], blue_noise=blue_noise)
    cg = scenes.apply(grp, sc)
    grp.set_option(OPT_TEMPORAL_AA, 1)
    grp.tick()
    with pytest.raises(Exception, match="TEMPORAL_AA"):
        grp.render_camera(cg)
    grp.set_option(OPT_TEMPORAL_AA, 0)
    grp.tick()
    grp.render_camera(cg)
    assert np.isfinite(grp.read_buffer(cg, "output")).all()
    one = _gpu_engine(blue_noise, False)
    c1 = scenes.apply(one, sc)
    one.tick()
    with pytest.raises(Exception, match="TEMPORAL_AA"):
        one.render_strips(c1)
    one.render_camera(c1)
    assert one.get_stat(STAT_TAA_RESOLVES) == 1


@pytest.mark.gpu
def test_antialiasing_on_device(blue_noise):
    """The anti-aliasing property on the device (product defaults): after 32 static frames of aa_edges the edge error against the
    8x8-supersampled option-off oracle render is at most half the option-off device frame's."""
    w, h, s = AA_W, AA_H, AA_S
    sc = scenes.aa_edges(w, h)
    res = {}
    for on in (False, True):
        e = _gpu_engine(blue_noise, False, taa=on)
        cam = scenes.apply(e, sc)
        for f in range(32):
            e.tick(); e.render_camera(cam)
        res[on] = e.read_buffer(cam, "output").reshape(h, w, 4)[..., :3].astype(np.float64)
    big = _aa_frames(blue_noise, False, 1, 0, w * s, h * s, first=16)[0][0]
    blk = big.reshape(h, s, w, s, 3)
    truth, edge = blk.mean((1, 3)), (blk.max((1, 3)) != blk.min((1, 3))).any(-1)
    err = {on: float(np.abs(res[on] - truth)[edge].mean()) for on in res}
    print(f"device aa_edges: edge error off {err[False]:.4f}, on {err[True]:.4f}, ratio {err[True] / err[False]:.3f}")
    assert err[True] <= 0.5 * err[False]
