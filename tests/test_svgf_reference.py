"""The denoiser passes (K20 reproject, K21 estimate_variance, K22 à-trous), frame composition and the Rgba8UnormSrgb store on the
device, pass by pass and pixel by pixel, against the float64 restatement in tests/ref64_svgf.py within its derived per-pixel bound
for the arithmetic tier that ran (strict IEEE, or the product default's SFU approximations + FMA).

The bit-parity tests compare the CUDA frame with the CPU oracle; these do not go through the oracle, and they see errors that stay
confined to a few pixels, which a whole-image relative L2 does not."""
import numpy as np
import pytest

from strolle_b200 import scenes
from tests import ref64_svgf as R
from tests.util import check_within, write_buffer

pytestmark = pytest.mark.gpu

P_REPROJECT, P_VARIANCE, P_WAVELET, P_COMPOSITION = 17, 18, 19, 20
SCENES = {"cornell": scenes.cornell, "demo_level": scenes.demo_level, "textured_room": scenes.textured_room}
DI_IO = [("stash", "prev_colors"), ("prev_colors", "stash"), ("stash", "curr_colors"), ("curr_colors", "stash"), ("stash", "curr_colors")]


@pytest.fixture(scope="module")
def gpu():
    import strolle_b200
    return strolle_b200


def _engine(gpu, blue_noise, strict, options=()):
    e = gpu.Engine(blue_noise=blue_noise, exact=strict)
    for k, v in options:
        e.set_option(k, v)
    return e


class Frame:
    """Steps through one frame's schedule and reads buffers as (H, W, 4)."""

    def __init__(self, e, cam, w, h):
        self.e, self.cam, self.w, self.h = e, cam, w, h
        self.sched = e.frame_schedule(cam)
        self.done = -1

    def read(self, name):
        return self.e.read_buffer(self.cam, name).reshape(self.h, self.w, 4)

    def write(self, name, a):
        write_buffer(self.e, self.cam, name, np.asarray(a, dtype=np.float32))

    def steps(self, pass_id):
        return [i for i, p in enumerate(self.sched) if p == pass_id]

    def run_to(self, last):
        if last > self.done:
            self.e.render_range(self.cam, self.done + 1, last)
            self.done = last


def _move(e, cam, scene, f):
    c = scene["camera"]
    t = np.asarray(c["transform"], dtype=np.float32).copy().reshape(16)
    t[12] += np.float32(0.011 * f); t[13] += np.float32(0.005 * f)
    e.update_camera(cam, c["mode"], c["denoise"], c["ref_depth"], c["w"], c["h"], t, c["projection"])


def _check_frame(fr, f, bn, fast, paired, ratios, tag, inject=None):
    """One frame, pass by pass.  `inject(stage, fr)` may overwrite the inputs of a stage right before it runs."""
    cur = "b" if f % 2 == 1 else "a"
    old = "a" if cur == "b" else "b"
    rp_steps, var_steps, wav_steps, comp_steps = fr.steps(P_REPROJECT), fr.steps(P_VARIANCE), fr.steps(P_WAVELET), fr.steps(P_COMPOSITION)
    fr.run_to(rp_steps[0] - 1)
    if inject:
        inject("K20", fr)
    sm = fr.read(f"prim_surface_map_{cur}")
    # surface_nd, which K21 / K22 read, is the f32 decode of the surface map
    nd = fr.read("surface_nd")
    n64, d32 = R.surface(sm)
    assert (nd[..., 3] == d32).all(), f"{tag} f{f}: surface_nd depth"
    live = d32 != 0
    assert (np.abs(nd[..., :3] - n64)[live] <= R.NORMAL_DECODE_ERR).all(), f"{tag} f{f}: surface_nd normal"
    src = {n: fr.read(n) for n in ("di_diff_samples", "gi_diff_samples", "reprojection_map", "di_diff_prev_colors", "gi_diff_prev_colors",
                                   f"di_diff_moments_{old}", f"gi_diff_moments_{old}", f"di_diff_moments_{cur}", f"gi_diff_moments_{cur}")}
    fr.run_to(rp_steps[-1])
    for sig in ("di", "gi"):
        r = R.reproject(src[f"{sig}_diff_samples"], sm, src["reprojection_map"], src[f"{sig}_diff_prev_colors"], src[f"{sig}_diff_moments_{old}"])
        want_m = np.where(r["sky"][..., None], src[f"{sig}_diff_moments_{cur}"], r["moment"])
        ratios["K20"] = max(ratios.get("K20", 0), check_within(fr.read(f"{sig}_diff_moments_{cur}"), want_m, r["b_moment"], f"{tag} f{f} K20 {sig} moments"))
        ratios["K20"] = max(ratios["K20"], check_within(fr.read(f"{sig}_diff_curr_colors"), r["color"], r["b_color"], f"{tag} f{f} K20 {sig} colours"))
    if inject:
        inject("K21", fr)
        sm = fr.read(f"prim_surface_map_{cur}")
    cols = {s: fr.read(f"{s}_diff_curr_colors") for s in ("di", "gi")}
    moms = {s: fr.read(f"{s}_diff_moments_{cur}") for s in ("di", "gi")}
    fr.run_to(var_steps[0])
    v = R.estimate_variance(sm, cols, moms, fast=fast)
    for sig in ("di", "gi"):
        key = f"K21 {'fast' if fast else 'strict'}"
        ratios[key] = max(ratios.get(key, 0), check_within(fr.read(f"{sig}_diff_stash"), v[sig], v["b_" + sig], f"{tag} f{f} K21 {sig}"))
    # K22: iterations that hand over through the private {DI, GI} records are compared as one span
    first_paired = {0: 5, 1: 4, 2: 3}[paired] if fast else 5
    spans = [[i] for i in range(5)] if first_paired == 5 else [[i] for i in range(first_paired - 1)] + [list(range(first_paired - 1, 5))]
    for span in spans:
        if inject:
            inject(f"K22 {span[0]}", fr)
            sm = fr.read(f"prim_surface_map_{cur}")
        src_name, dst_name = DI_IO[span[0]][0], DI_IO[span[-1]][1]
        di_in, gi_in = fr.read(f"di_diff_{src_name}"), fr.read(f"gi_diff_{src_name}")
        gi_before = fr.read(f"gi_diff_{dst_name}")
        fr.run_to(wav_steps[span[-1]])
        r = R.wavelet_chain(sm, di_in, gi_in, span, f, bn, fast=fast)
        gi_want = np.where(r["sky"][..., None], gi_before, r["gi"])        # a sky centre does not write GI
        key = f"K22 {span[0]}-{span[-1]} {'fast' if fast else 'strict'}"
        ratios[key] = max(ratios.get(key, 0), check_within(fr.read(f"di_diff_{dst_name}"), r["di"], r["b_di"], f"{tag} f{f} K22 {span} di"))
        ratios[key] = max(ratios[key], check_within(fr.read(f"gi_diff_{dst_name}"), gi_want, r["b_gi"], f"{tag} f{f} K22 {span} gi"))
    if inject:
        inject("composition", fr)
    ins = {n: fr.read(n) for n in (f"prim_gbuffer_d0_{cur}", f"prim_gbuffer_d1_{cur}", "di_diff_curr_colors", "gi_diff_curr_colors",
                                   "di_spec_samples", "gi_spec_samples", "ref_colors")}
    fr.run_to(comp_steps[-1])
    col, b = R.compose(0, ins[f"prim_gbuffer_d0_{cur}"], ins[f"prim_gbuffer_d1_{cur}"], ins["di_diff_curr_colors"], ins["gi_diff_curr_colors"],
                       ins["di_spec_samples"], ins["gi_spec_samples"], ins["ref_colors"])
    out = fr.read("output")
    ratios["composition"] = max(ratios.get("composition", 0), check_within(out[..., :3], col, b, f"{tag} f{f} composition"))
    assert (out[..., 3] == 1).all()
    assert fr.done == len(fr.sched) - 1


def _run(gpu, blue_noise, scene, strict, frames=6, moves=(3, 5), options=(), inject=None, tag=""):
    from strolle_b200.engine import OPT_WAVELET_PAIRED
    e = _engine(gpu, blue_noise, strict, options)
    cam = scenes.apply(e, scene)
    w, h = scene["camera"]["w"], scene["camera"]["h"]
    paired = dict(options).get(OPT_WAVELET_PAIRED, 1)
    ratios = {}
    for f in range(1, frames + 1):
        if f in moves:
            _move(e, cam, scene, f)
        e.tick()
        _check_frame(Frame(e, cam, w, h), f, blue_noise, not strict, paired, ratios, tag, inject)
    return e, cam, ratios


@pytest.mark.parametrize("size", [(224, 126), (67, 45), (37, 29)])
@pytest.mark.parametrize("scene_name", ["cornell", "demo_level", "textured_room"])
@pytest.mark.parametrize("strict", [True, False], ids=["strict", "default"])
def test_svgf_passes_within_float64_bound(gpu, blue_noise, strict, scene_name, size):
    """Every pixel and channel of K20, K21, each K22 iteration (or paired span) and the composition within the derived bound, frames
    1-6 (history below and past 4), camera moving on frames 3 and 5 (K20's bilinear path), on sizes narrower than stride 16's reach."""
    from strolle_b200.engine import STAT_WAVELET_TILED_ERRORS, STAT_WAVELET_TILED_LAUNCHES, STAT_VARIANCE_TILED_LAUNCHES
    e, _, ratios = _run(gpu, blue_noise, SCENES[scene_name](*size), strict, tag=f"{scene_name} {size}")
    assert e.get_stat(STAT_WAVELET_TILED_ERRORS) == 0
    if not strict:   # the product default: K21 and K22 tile-staged, strides 8-16 handed over through the paired records
        assert e.get_stat(STAT_VARIANCE_TILED_LAUNCHES) > 0 and e.get_stat(STAT_WAVELET_TILED_LAUNCHES) > 0
        assert "K22 3-4 fast" in ratios, ratios
    print(f"\n{scene_name} {size} {'strict' if strict else 'default'}: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(ratios.items())))


def _variants():
    from strolle_b200 import engine as E
    out = []
    for fuse in (0, 1):
        for vt in (0, 1):
            out.append(((E.OPT_FUSE_REPROJECT, fuse), (E.OPT_VARIANCE_TILED, vt), (E.OPT_WAVELET_TILED, 0), (E.OPT_WAVELET_PAIRED, 0)))
    for cfg in range(4):
        out.append(((E.OPT_WAVELET_TILED, 31), (E.OPT_WAVELET_TILE_CFG, cfg * 0x11111), (E.OPT_WAVELET_PAIRED, 0)))
    for paired in (1, 2):
        for tiled in (0, 31):
            out.append(((E.OPT_WAVELET_TILED, tiled), (E.OPT_WAVELET_PAIRED, paired)))
    return out


@pytest.mark.parametrize("variant", range(12))
def test_svgf_kernel_variants_within_bound(gpu, blue_noise, variant):
    """K20 fused pair and split, K21 gather and tiled, K22 gather, tile-staged with every tile shape for every iteration, and paired
    records 1 / 2 (gather and tiled producers), fast tier, Cornell 67x45 (ragged tiles, sky) over 5 frames with a moving camera."""
    from strolle_b200.engine import STAT_WAVELET_TILED_ERRORS, STAT_WAVELET_TILED_LAUNCHES, OPT_WAVELET_TILED, OPT_WAVELET_PAIRED
    opts = _variants()[variant]
    e, _, ratios = _run(gpu, blue_noise, scenes.cornell(67, 45), False, frames=5, moves=(2, 4), options=opts, tag=f"variant {opts}")
    o = dict(opts)
    assert e.get_stat(STAT_WAVELET_TILED_ERRORS) == 0
    tiled, paired = o.get(OPT_WAVELET_TILED, 15), o.get(OPT_WAVELET_PAIRED, 1)
    first_paired = {0: 5, 1: 4, 2: 3}[paired]
    planar_tiled = sum(1 for i in range(5) if (tiled >> i) & 1 and i < first_paired)
    assert e.get_stat(STAT_WAVELET_TILED_LAUNCHES) == 5 * planar_tiled


def test_svgf_fast_tier_is_not_strict(gpu, blue_noise):
    """The product default's K22 really runs the approximate arithmetic: the same inputs through the strict kernel give different
    bits somewhere (so the fast-tier runs above cannot be strict runs in disguise)."""
    from strolle_b200.engine import OPT_SVGF_FAST_MATH
    scene = scenes.cornell(67, 45)
    e = _engine(gpu, blue_noise, False)
    cam = scenes.apply(e, scene)
    for _ in range(2):
        e.tick(); e.render_camera(cam)
    e.tick()
    fr = Frame(e, cam, 67, 45)
    k = fr.steps(P_WAVELET)[0]
    fr.run_to(k - 1)
    before = fr.read("di_diff_prev_colors")
    fr.run_to(k)
    fast = fr.read("di_diff_prev_colors")
    fr.write("di_diff_prev_colors", before)
    e.set_option(OPT_SVGF_FAST_MATH, 0)
    e.render_range(cam, k, k)
    strict = fr.read("di_diff_prev_colors")
    assert (fast.view(np.uint32) != strict.view(np.uint32)).any()


def test_svgf_1080p_product_default(gpu, blue_noise):
    """One product-default 1920x1080 frame, every pass within its bound."""
    from strolle_b200.engine import STAT_WAVELET_TILED_ERRORS
    e, _, ratios = _run(gpu, blue_noise, scenes.cornell(1920, 1080), False, frames=1, moves=(), tag="1080p")
    assert e.get_stat(STAT_WAVELET_TILED_ERRORS) == 0


# ---- edge inputs ------------------------------------------------------------------------------------------------------------

def _oct_encode(n):
    """Normal::encode (normal.rs) in f64, stored as f32."""
    n = np.asarray(n, dtype=np.float64)
    n = n / np.abs(n).sum(-1, keepdims=True)
    xy = n[..., :2].copy()
    neg = n[..., 2] < 0
    t = 1.0 - np.abs(n[..., ::-1][..., 1:3])       # (1 - |y|, 1 - |x|)
    xy = np.where(neg[..., None], np.copysign(t, n[..., :2]), xy)
    return (xy * 0.5 + 0.5).astype(np.float32)


class Edges:
    """Writes edge-case contents into the buffers a stage reads (sizes, strides and indices stay what the engine allocated)."""

    def __init__(self, w, h, seed, f_cur, all_sky=False):
        self.w, self.h, self.rng = w, h, np.random.RandomState(seed)
        self.cur = f_cur
        self.all_sky = all_sky

    def surface(self, depth_sigma):
        rng, h, w = self.rng, self.h, self.w
        D = np.float32(2.0)
        leeway = np.float32(D * np.float32(depth_sigma))
        cut = np.float32(D + leeway)
        choices = np.array([D, np.nextafter(cut, np.float32(0)), cut, np.nextafter(cut, np.float32(9)), D * np.float32(1.01), np.float32(0.0)],
                           dtype=np.float32)
        depth = np.where(rng.rand(h, w) < 0.6, D, choices[rng.randint(0, len(choices), (h, w))]).astype(np.float32)
        if self.all_sky:
            depth[:] = 0; depth[h // 2, w // 2] = D
        nrm = np.tile(np.array([0.0, 0.0, 1.0]), (h, w, 1))
        k = rng.randint(0, 5, (h, w))
        nrm[k == 1] = (1.0, 0.0, 0.0)                  # 90 degrees
        nrm[k == 2] = (0.0, 0.0, -1.0)                 # 180 degrees
        nrm[k == 3] = (0.3, -0.2, 0.93)
        sm = np.zeros((h, w, 4), np.float32)
        sm[..., 0:2] = _oct_encode(nrm)
        sm[..., 2] = depth
        sm[..., 3] = 0.5
        nd = np.zeros((h, w, 4), np.float32)
        nd[..., :3] = np.where((depth != 0)[..., None], R.decode_normal(sm), 0.0).astype(np.float32)
        nd[..., 3] = depth
        return sm, nd

    def colors(self, variance=True):
        rng, h, w = self.rng, self.h, self.w
        c = rng.uniform(0, 2, (h, w, 4)).astype(np.float32)
        k = rng.randint(0, 14, (h, w))
        c[k == 1, :3] = 0.0                                           # luma 0
        c[k == 2, :3] = np.float32(1e-40)                             # denormal luma
        c[k == 3, :3] = np.float32(1e6)                               # very large luma
        c[k == 4, 1] = np.nan                                         # NaN sample
        c[k == 5, 0] = np.inf
        c[k == 6, 2] = -np.inf
        c[k == 7, :3] = np.float32(3e-39)                             # just below FLT_MIN
        if variance:
            c[k == 8, 3] = 0.0
            c[k == 9, 3] = np.float32(1e-41)
            c[k == 10, 3] = np.float32(1.5)                           # sqrt(var) > 1: sigma clamps
        return c

    def inject(self, stage, fr):
        cur = self.cur
        if stage == "K20":
            sm, nd = self.surface(0.2)
            fr.write(f"prim_surface_map_{cur}", sm); fr.write("surface_nd", nd)
            rng, h, w = self.rng, self.h, self.w
            ys, xs = np.mgrid[0:h, 0:w].astype(np.float32)
            px, py = xs.copy(), ys.copy()
            k = rng.randint(0, 8, (h, w))
            px[k == 1] += np.float32(0.25); py[k == 1] += np.float32(0.5)             # fractional
            px[k == 2] = np.float32(-0.375)                                          # x in (-1, 0)
            px[k == 3] = np.float32(w - 1) + np.float32(0.5)                         # last column, fractional: ceil reads x = w
            py[k == 4] = np.float32(h - 1) + np.float32(0.75)                        # last row, fractional
            px[k == 5] = np.float32(w - 1); py[k == 5] = np.float32(h - 1)           # exact corner
            px[k == 6] += np.float32(0.5)                                            # half: fract 0.5
            rp = np.zeros((h, w, 4), np.float32)
            rp[..., 0], rp[..., 1] = px, py
            rp[..., 2] = np.where(rng.rand(h, w) < 0.15, 0.0, rng.uniform(0.1, 1, (h, w))).astype(np.float32)   # confidence 0
            rp[..., 3] = rng.randint(0, 16, (h, w)).astype(np.uint32).view(np.float32)                          # validity 0-15
            fr.write("reprojection_map", rp)
            old = "a" if cur == "b" else "b"
            for sig in ("di", "gi"):
                s = rng.uniform(0, 2, (h, w, 4)).astype(np.float32)
                s[..., 3] = np.where(rng.rand(h, w) < 0.15, 0.0, 1.0)                     # sample.w == 0
                fr.write(f"{sig}_diff_samples", s)
                fr.write(f"{sig}_diff_prev_colors", rng.uniform(0, 2, (h, w, 4)).astype(np.float32))
                m = rng.uniform(0, 1, (h, w, 4)).astype(np.float32)
                m[..., 0] = rng.randint(0, 17, (h, w))                                     # history 0-16: cap at 16
                fr.write(f"{sig}_diff_moments_{old}", m)
        elif stage == "K21":
            sm, nd = self.surface(0.2)
            fr.write(f"prim_surface_map_{cur}", sm); fr.write("surface_nd", nd)
            for sig in ("di", "gi"):
                fr.write(f"{sig}_diff_curr_colors", self.colors(variance=False))
                m = self.rng.uniform(0, 1, (self.h, self.w, 4)).astype(np.float32)
                m[..., 0] = np.where(self.rng.rand(self.h, self.w) < 0.5, 3.0, 4.0)      # history 3 and 4
                fr.write(f"{sig}_diff_moments_{cur}", m)
        elif stage.startswith("K22"):
            it = int(stage.split()[1])
            sm, nd = self.surface(np.float32(0.33) / np.float32(1 + it))
            fr.write(f"prim_surface_map_{cur}", sm); fr.write("surface_nd", nd)
            src = DI_IO[it][0]
            for sig in ("di", "gi"):
                fr.write(f"{sig}_diff_{src}", self.colors())
        elif stage == "composition":
            pass


@pytest.mark.parametrize("all_sky", [False, True], ids=["mixed", "all_sky_but_one"])
@pytest.mark.parametrize("strict", [True, False], ids=["strict", "default"])
@pytest.mark.parametrize("paired", [0, 1, 2])
def test_svgf_edge_inputs_within_bound(gpu, blue_noise, strict, paired, all_sky):
    """Edge contents injected before each pass: depth differences just below / at / above the cut-off, normals at 0, 90 and 180
    degrees, sky centres and taps (and a frame that is all sky but one pixel), K21 history 3 and 4, variance 0 / denormal / > 1,
    luma 0 / denormal / 1e6, NaN and +-inf in a tap's colour, K20 validity masks 0-15, exact and fractional previous positions
    (x in (-1, 0), the last column and row), confidence 0 and sample.w 0."""
    from strolle_b200.engine import OPT_WAVELET_PAIRED
    if strict and paired:
        pytest.skip("the strict tier has no paired records")
    w, h = 37, 29
    scene = scenes.cornell(w, h)
    e = _engine(gpu, blue_noise, strict, [(OPT_WAVELET_PAIRED, paired)])
    cam = scenes.apply(e, scene)
    ratios = {}
    for f in range(1, 4):
        e.tick()
        ed = Edges(w, h, 100 * f + paired, "b" if f % 2 == 1 else "a", all_sky)
        _check_frame(Frame(e, cam, w, h), f, blue_noise, not strict, paired, ratios, f"edges f{f}", ed.inject)
    print("\nedges: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(ratios.items())))


# ---- composition and sRGB ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("mode", range(7))
def test_composition_modes_within_bound(gpu, blue_noise, mode):
    """frame_composition::fs for every camera mode on injected G-buffer and signal buffers: mode 0 on surface and sky pixels,
    base colour (b / 255)^2.2 from the packed bytes, mode 6 divides by w."""
    w, h = 53, 31
    scene = scenes.cornell(w, h, mode=mode)
    e = _engine(gpu, blue_noise, False)
    cam = scenes.apply(e, scene)
    e.tick()
    fr = Frame(e, cam, w, h)
    n = len(fr.sched)
    fr.run_to(n - 2)
    rng = np.random.RandomState(mode)
    cur = "b"
    d0 = rng.uniform(0.5, 4, (h, w, 4)).astype(np.float32)
    d0[rng.rand(h, w) < 0.3, 0] = 0.0                                                    # sky
    d1 = rng.uniform(0, 3, (h, w, 4)).astype(np.float32)
    d1[..., 3] = rng.randint(0, 2 ** 32, (h, w), dtype=np.uint64).astype(np.uint32).view(np.float32)
    sig = {n_: rng.uniform(0, 2, (h, w, 4)).astype(np.float32) for n_ in ("dd", "gd", "ds", "gs", "rc")}
    sig["rc"][..., 3] = rng.uniform(0.5, 64, (h, w)).astype(np.float32)
    fr.write(f"prim_gbuffer_d0_{cur}", d0); fr.write(f"prim_gbuffer_d1_{cur}", d1)
    for name in ("di_diff_curr_colors", "di_diff_samples"):
        fr.write(name, sig["dd"])
    for name in ("gi_diff_curr_colors", "gi_diff_samples"):
        fr.write(name, sig["gd"])
    fr.write("di_spec_samples", sig["ds"]); fr.write("gi_spec_samples", sig["gs"]); fr.write("ref_colors", sig["rc"])
    fr.run_to(n - 1)
    assert fr.sched[-1] == P_COMPOSITION
    col, b = R.compose(mode, d0, d1, sig["dd"], sig["gd"], sig["ds"], sig["gs"], sig["rc"])
    out = fr.read("output")
    check_within(out[..., :3], col, b, f"mode {mode}")
    assert (out[..., 3] == 1).all()


def _srgb_inputs():
    f = np.float32
    specials = np.array([-np.inf, -1.0, -0.0, 0.0, 1e-45, 1e-40, 1.1754942e-38, 1.0, np.nextafter(f(1), f(2)), 1e30, np.inf, np.nan], f)
    th = f(0.0031308)
    near = [th]
    for _ in range(4):
        near += [np.nextafter(near[-1], f(1))]
    x = th
    for _ in range(4):
        x = np.nextafter(x, f(0)); near.append(x)
    # f32 preimages of every byte's rounding boundary (k + 0.5) / 255 of the encoded value, +-4 ulp around each
    e = (np.arange(256) + 0.5) / 255.0
    pre = np.where(e <= 12.92 * 0.0031308, e / 12.92, ((e + 0.055) / 1.055) ** 2.4)
    pre = pre[pre <= 1.0].astype(f)
    around = [pre]
    up, dn = pre.copy(), pre.copy()
    for _ in range(4):
        up = np.nextafter(up, f(2)); dn = np.nextafter(dn, f(-1))
        around += [up, dn]
    uni = np.random.RandomState(7).uniform(0, 1, 10 ** 6).astype(f)
    return np.concatenate([specials, np.array(near, f), np.concatenate(around), uni]).astype(f)


@pytest.mark.parametrize("async_output", [0, 1], ids=["blocking", "async"])
def test_rgba8_srgb_store(gpu, blue_noise, async_output):
    """copy_output(Rgba8UnormSrgb) of an injected `output`: specials (-inf, -1, -0, 0, denormals, 1, 1 + ulp, 1e30, +inf, NaN -> 0),
    0.0031308 and its f32 neighbours, +-4 ulp around the f32 preimage of every byte's rounding boundary and 10^6 uniform values.
    Bytes equal the f64 encoding exactly except within the derived window around a .5 boundary, where they may differ by one;
    alpha is 255."""
    import torch
    from strolle_b200.engine import FORMAT_RGBA8_SRGB, OPT_ASYNC_OUTPUT
    vals = _srgb_inputs()
    w, h = 640, 480
    per = w * h * 3
    e = _engine(gpu, blue_noise, False, [(OPT_ASYNC_OUTPUT, async_output)])
    cam = scenes.apply(e, scenes.cornell(w, h))
    e.tick(); e.render_camera(cam)
    loose = 0
    for k in range(0, vals.size, per):
        chunk = vals[k:k + per]
        rgb = np.zeros(per, np.float32)
        rgb[:chunk.size] = chunk
        out = np.ones((h, w, 4), np.float32)
        out[..., :3] = rgb.reshape(h, w, 3)
        write_buffer(e, cam, "output", out)
        pinned = torch.zeros((h, w, 4), dtype=torch.uint8, pin_memory=True)
        host = pinned.numpy()
        e.copy_output(cam, host, FORMAT_RGBA8_SRGB)
        e.synchronize()
        assert (host[..., 3] == 255).all()
        got = host[..., :3].reshape(-1)[:chunk.size].astype(np.int64)
        want, t, dt = R.srgb_encode(chunk)
        near = np.abs(t - np.round(t)) <= dt
        exact_ok = got == want
        assert (exact_ok | (near & (np.abs(got - want) <= 1))).all(), \
            f"bytes differ outside the rounding window: {chunk[~exact_ok & ~near][:8].tolist()} -> {got[~exact_ok & ~near][:8].tolist()} vs {want[~exact_ok & ~near][:8].tolist()}"
        loose += int((~exact_ok).sum())
    print(f"\nsRGB: {vals.size} values, {loose} off by one inside the window")
