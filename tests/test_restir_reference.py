"""The DI spatial merge (K9) and DI resolving (K10) on the device, pass by pass and value by value, against the float64 restatement in
tests/ref64_restir.py within its derived bound for the arithmetic tier that ran (strict IEEE, or the fast-shading build: FMA
contraction, div.full / sqrt.approx).  Also the fast build's elementary functions against the constants a bound on them assumes.

The bit-parity tests compare the CUDA frame with the CPU oracle, which came from the same reading of the reference; these do not go
through the oracle, and unlike a whole-image relative L2 they see an error confined to a few pixels (a light's falloff near its range
edge, a GGX highlight, a merge whose M or w is off)."""
import numpy as np
import pytest

from strolle_b200 import scenes
from tests import ref64_restir as Q
from tests.util import Frame, check_within, write_buffer

pytestmark = pytest.mark.gpu

P_DI_SPATIAL_SAMPLE, P_DI_RESOLVING = 5, 6
SEED_BASE = 0xC0FFEE
SCENES = {"cornell": scenes.cornell, "demo_level": scenes.demo_level, "textured_room": scenes.textured_room,
          "cornell_spots": lambda w, h: scenes.cornell_spots(w, h)}
# undecided decisions allowed per pass, as a fraction of the values checked.  None were seen in the scene runs on an H100 (24 runs, both
# tiers); the injected M = 1e6 / w = 1e6 reservoirs put 3.6 % of K9's merges inside the bound of `rng W < weight` (W dominated by the
# huge weight, the other weight below its rounding), hence the looser limit there.
UNDECIDED_MAX = 0.001
UNDECIDED_MAX_EDGES = 0.1


@pytest.fixture(scope="module")
def gpu():
    import strolle_b200
    return strolle_b200


def _engine(gpu, blue_noise, strict, fused):
    from strolle_b200.engine import OPT_FUSED_PASSES
    e = gpu.Engine(blue_noise=blue_noise, exact=strict)
    e.set_option(OPT_FUSED_PASSES, int(fused))
    return e


class Chain:
    """Drives one camera frame by frame and checks K9 / K10 as they run."""

    def __init__(self, gpu, blue_noise, scene, strict, fused):
        self.e = _engine(gpu, blue_noise, strict, fused)
        self.scene = scene
        self.cam = scenes.apply(self.e, scene)
        c = scene["camera"]
        self.w, self.h = c["w"], c["h"]
        self.t = np.asarray(c["transform"], np.float32).reshape(16).copy()
        self.fast = not strict
        self.stats = {"K9": [0.0, 0, 0], "K10": [0.0, 0, 0]}
        self.k9_tight = [0, 0]     # (tightly bounded, finite nonzero) m and w of the merged pairs
        self.bounds = []
        self.f = 0

    def move(self, f):
        c = self.scene["camera"]
        self.t[12] += np.float32(0.013 * f); self.t[13] += np.float32(0.004 * f)
        self.e.update_camera(self.cam, c["mode"], c["denoise"], c["ref_depth"], self.w, self.h, self.t, c["projection"])

    def frame(self, inject_k9=None, inject_k10=None):
        e, cam, w, h = self.e, self.cam, self.w, self.h
        self.f += 1
        f = self.f
        e.tick()
        fr = Frame(e, cam, w, h)
        cur = "b" if f % 2 == 1 else "a"
        k9 = fr.steps(P_DI_SPATIAL_SAMPLE)
        if k9:   # unfused schedule: K9 reads K8's visibility texels from di_diff_stash
            fr.run_to(k9[0] - 1)
            if inject_k9:
                inject_k9(fr)
            r1, stash = e.read_buffer(cam, "di_reservoirs_1"), fr.read("di_diff_stash")
            fr.run_to(k9[0])
            r = Q.di_spatial_sample(r1, stash, Q.dispatch_seed(SEED_BASE, f, P_DI_SPATIAL_SAMPLE), f, w, h, self.fast)
            ratio, und, merged = Q.check_spatial_sample(e.read_buffer(cam, "di_reservoirs_2"), r1, r, f"f{f} K9")
            s = self.stats["K9"]
            self.stats["K9"] = [max(s[0], ratio), s[1] + und, s[2] + merged]
            frac, n = Q.spatial_sample_tight(r)
            self.k9_tight = [self.k9_tight[0] + round(frac * n), self.k9_tight[1] + n]
        k10 = fr.steps(P_DI_RESOLVING)[0]
        fr.run_to(k10 - 1)
        if inject_k10:
            inject_k10(fr, cur)
        d0, d1 = fr.read(f"prim_gbuffer_d0_{cur}"), fr.read(f"prim_gbuffer_d1_{cur}")
        r2 = e.read_buffer(cam, "di_reservoirs_2")
        fr.run_to(k10)
        res0 = e.read_buffer(cam, "di_reservoirs_0")
        r = Q.di_resolving(Q.ndc_to_world(self.t, self.scene["camera"]["projection"]), w, h, d0, d1, e.read_scene("lights"), r2, res0, self.fast)
        ratio, und, b = Q.check_resolving(fr.read("di_diff_samples"), fr.read("di_spec_samples"), res0, r, f"f{f} K10", check_within)
        s = self.stats["K10"]
        self.stats["K10"] = [max(s[0], ratio), s[1] + und, s[2] + int(r["some"].sum())]
        self.bounds.append((b, r["some"]))
        fr.run_to(len(fr.sched) - 1)
        return r

    def report(self, tag, limit=UNDECIDED_MAX):
        s9, s10 = self.stats["K9"], self.stats["K10"]
        print(f"\n{tag}: K9 ratio {s9[0]:.3g} undecided {s9[1]}/{s9[2]}; K10 ratio {s10[0]:.3g} undecided specular {s10[1]}/{s10[2]}")
        assert s9[1] <= limit * max(s9[2], 1) and s10[1] <= limit * max(s10[2], 1)


def _run(gpu, blue_noise, scene, strict, fused, frames=13, moves=(3, 5, 8, 11)):
    ch = Chain(gpu, blue_noise, scene, strict, fused)
    for f in range(1, frames + 1):
        if f in moves:
            ch.move(f)
        if f == 4:
            ch.e.insert_light(9001, scenes.LIGHT_POINT, scenes.point_light((0.2, 1.0, 0.3), 0.08, (3.0, 2.0, 1.0), 6.0))
        if f == 7:
            ch.e.insert_light(9001, scenes.LIGHT_POINT, scenes.point_light((-0.3, 0.8, 0.1), 0.08, (3.0, 2.0, 1.0), 6.0))
        if f == 10:
            ch.e.remove_light(9001)
        ch.frame()
    return ch


@pytest.mark.parametrize("size", [(224, 126), (67, 45), (37, 29)])
@pytest.mark.parametrize("scene_name", ["cornell", "demo_level", "textured_room", "cornell_spots"])
@pytest.mark.parametrize("strict", [True, False], ids=["strict", "fast"])
def test_di_merge_and_resolve_within_float64_bound(gpu, blue_noise, strict, scene_name, size):
    """K9 and K10 in the unfused schedule, every pair / pixel, frames 1-13 (both GI cycles) with the camera moving and a light
    inserted, moved and removed; 67x45 leaves columns outside the half grid, 37x29 is smaller than the 128 px tap radius."""
    ch = _run(gpu, blue_noise, SCENES[scene_name](*size), strict, fused=False)
    assert ch.stats["K9"][2] > 0 and 0 < ch.stats["K10"][0] <= 1
    ch.report(f"{scene_name} {size} {'strict' if strict else 'fast'}")
    # the bound is not vacuous: most values are bounded tightly, and some error uses a visible part of its bound
    b, some = ch.bounds[-1]
    frac, n = Q.tight_fraction(list(b), some)
    assert n > 0 and frac >= 0.99, frac
    assert ch.k9_tight[1] > 0 and ch.k9_tight[0] >= 0.99 * ch.k9_tight[1], ch.k9_tight
    assert ch.stats["K10"][0] > 1e-3 and ch.stats["K9"][0] > 1e-3


@pytest.mark.parametrize("scene_name", ["cornell", "demo_level"])
def test_di_resolve_product_default_within_bound(gpu, blue_noise, scene_name):
    """The product default (fast build, fused passes): K10 still runs as its own launch and is checked against the bound."""
    ch = _run(gpu, blue_noise, SCENES[scene_name](224, 126), strict=False, fused=True)
    assert ch.stats["K9"][2] == 0 and ch.stats["K10"][2] > 0
    ch.report(f"{scene_name} product default")


def test_di_resolve_1080p_product_default(gpu, blue_noise):
    ch = _run(gpu, blue_noise, scenes.cornell(1920, 1080), strict=False, fused=True, frames=2, moves=())
    ch.report("1080p product default")


# ---- injected edge inputs ------------------------------------------------------------------------------------------------------

def _gbuffer_edges(seed, ch):
    """Rewrites the surface bytes of the G-buffer before K10: metallic 0 / 255, roughness byte 0 (the 0.089^2 clamp), reflectance
    0 / 255, and the normal along the view direction at minimum roughness (GGX's (n.h a^2 - n.h) n.h + 1 cancellation)."""
    def inject(fr, cur):
        rng = np.random.RandomState(seed)
        d0 = fr.read(f"prim_gbuffer_d0_{cur}").copy()
        bits = d0[..., 3].view(np.uint32).copy()
        m, r, f = bits & 0xFF, (bits >> 8) & 0xFF, (bits >> 16) & 0xFF
        k = rng.randint(0, 6, bits.shape)
        m = np.where(k == 1, 0, np.where(k == 2, 255, m)); r = np.where(k == 3, 0, r)
        f = np.where(k == 4, 0, np.where(k == 5, 255, f))
        mirror = rng.rand(*bits.shape) < 0.1
        m = np.where(mirror, 255, m); r = np.where(mirror, 0, r)
        d0[..., 3] = ((bits & 0xFF000000) | m | (r << 8) | (f << 16)).astype(np.uint32).view(np.float32)
        o, d = Q.camera_ray(Q.ndc_to_world(ch.t, ch.scene["camera"]["projection"]), fr.w, fr.h, False)
        n = -d.v
        n = n / np.abs(n).sum(-1, keepdims=True)
        xy = np.where((n[..., 2] < 0)[..., None], np.copysign(1.0 - np.abs(n[..., ::-1][..., 1:3]), n[..., :2]), n[..., :2])
        enc = (xy * 0.5 + 0.5).astype(np.float32)
        live = d0[..., 0] != 0
        d0[..., 1:3] = np.where((mirror & live)[..., None], enc, d0[..., 1:3])
        fr.write(f"prim_gbuffer_d0_{cur}", d0)
    return inject


def _reservoir_edges(seed):
    """Rewrites di_reservoirs[1] before K9: M at 63, 64, 65 and 1e6, w at 0, a denormal and 1e6, pdf 0."""
    def inject(fr):
        rng = np.random.RandomState(seed)
        r = fr.e.read_buffer(fr.cam, "di_reservoirs_1").reshape(-1, 8).copy()
        live = r[:, 0] > 0
        k = rng.randint(0, 9, len(r))
        r[:, 0] = np.where(live & (k == 1), 63, np.where(live & (k == 2), 64, np.where(live & (k == 3), 65, np.where(live & (k == 4), 1e6, r[:, 0]))))
        r[:, 1] = np.where(live & (k == 5), 0, np.where(live & (k == 6), np.float32(1e-41), np.where(live & (k == 7), 1e6, r[:, 1])))
        r[:, 2] = np.where(live & (k == 8), 0, r[:, 2])
        write_buffer(fr.e, fr.cam, "di_reservoirs_1", r.astype(np.float32))
    return inject


def edge_lights(engine):
    """Lights at the edges of Light::radiance: one 2 mm above the floor (l^2 toward the 1e-4 floor of f_dist), one whose range ends
    inside the box (the smooth factor reaching 0), one of infinite range, and a narrow spot straight down (hits on its axis and across
    its cone edge)."""
    engine.insert_light(9101, scenes.LIGHT_POINT, scenes.point_light((0.1, 0.002, 0.2), 0.001, (0.05, 0.05, 0.05), 2.0))
    engine.insert_light(9102, scenes.LIGHT_POINT, scenes.point_light((-0.4, 1.0, -0.2), 0.05, (2.0, 1.0, 1.0), 0.9))
    engine.insert_light(9103, scenes.LIGHT_POINT, scenes.point_light((0.3, 1.5, 0.4), 0.05, (0.5, 0.8, 1.0), np.inf))
    engine.insert_light(9104, scenes.LIGHT_SPOT, scenes.spot_light((0.0, 1.7, 0.0), 0.02, (4.0, 4.0, 3.0), 10.0, (0.0, -1.0, 0.0), 0.15))


@pytest.mark.parametrize("strict", [True, False], ids=["strict", "fast"])
@pytest.mark.parametrize("scene_name", ["cornell", "cornell_spots"])
def test_di_edge_inputs_within_bound(gpu, blue_noise, strict, scene_name):
    """Edge contents injected before K9 (M at the cap region and far past it, w 0 / denormal / 1e6, pdf 0) and before K10 (metallic
    and reflectance bytes 0 / 255, roughness byte 0, normals along the view direction at minimum roughness), with the edge lights."""
    ch = Chain(gpu, blue_noise, SCENES[scene_name](67, 45), strict, fused=False)
    edge_lights(ch.e)
    for f in range(1, 6):
        ch.frame(_reservoir_edges(10 * f), _gbuffer_edges(10 * f + 1, ch))
    ch.report(f"edges {scene_name} {'strict' if strict else 'fast'}", UNDECIDED_MAX_EDGES)


def test_fast_shading_build_is_not_strict(gpu, blue_noise):
    """The fast-tier runs above really ran the fast build: the same inputs through the strict K9 and the strict K10 give different bits
    somewhere in each pass's output."""
    from strolle_b200.engine import OPT_SHADING_FAST_MATH
    e = _engine(gpu, blue_noise, False, False)
    cam = scenes.apply(e, scenes.cornell(67, 45))
    for _ in range(2):
        e.tick(); e.render_camera(cam)
    e.tick()
    fr = Frame(e, cam, 67, 45)
    k9, k10 = fr.steps(P_DI_SPATIAL_SAMPLE)[0], fr.steps(P_DI_RESOLVING)[0]
    fr.run_to(k9)                        # K9 reads di_reservoirs[1] and the stash, which it leaves as they were
    fast9 = e.read_buffer(cam, "di_reservoirs_2").copy()
    fr.run_to(k10)                       # K10 reads di_reservoirs[2] and the G-buffer, and writes neither
    fast10 = fr.read("di_spec_samples").copy(), fr.read("di_diff_samples").copy()
    e.set_option(OPT_SHADING_FAST_MATH, 0)
    e.render_range(cam, k10, k10)
    strict10 = fr.read("di_spec_samples"), fr.read("di_diff_samples")
    e.render_range(cam, k9, k9)
    strict9 = e.read_buffer(cam, "di_reservoirs_2")
    assert (fast9.view(np.uint32) != strict9.view(np.uint32)).any(), "K9"
    assert any((a.view(np.uint32) != b.view(np.uint32)).any() for a, b in zip(fast10, strict10)), "K10"


# ---- the fast build's elementary functions ------------------------------------------------------------------------------------

def test_fast_elementary_functions_within_assumed_constants(gpu, blue_noise):
    """sin / cos (__sincosf), exp (__expf), pow (__powf), sqrt (sqrt.approx) and division (div.full) of the fast-shading build, measured
    on the argument ranges the ReSTIR kernels use, within the constants a bound on them assumes (tests/ref64_restir.py)."""
    e = gpu.Engine(blue_noise=blue_noise)
    rng = np.random.RandomState(3)
    x = np.concatenate([np.linspace(0, 2 * np.pi, 200001), rng.uniform(0, 2 * np.pi, 10 ** 6)]).astype(np.float32)
    x64 = x.astype(np.float64)
    err_s = np.abs(e.device_math("sin_fast", x) - np.sin(x64)).max()
    err_c = np.abs(e.device_math("cos_fast", x) - np.cos(x64)).max()
    xe = np.concatenate([np.linspace(-100, 0, 200001), rng.uniform(-20, 0, 10 ** 6)]).astype(np.float32)
    xe64 = xe.astype(np.float64)
    got = e.device_math("exp_fast", xe).astype(np.float64)
    want = np.exp(xe64)
    ok = want > 1e-37
    rel_e = (np.abs(got - want) / want - 2 * Q.U * np.abs(xe64) * np.log2(np.e))[ok].max()
    base = rng.uniform(1e-4, 1, 10 ** 6).astype(np.float32)
    expo = rng.choice(np.array([2.2, 1 / 2.4, 2.4, 1 / 2.2, 0.5, 4.0, 1.7], np.float32), 10 ** 6)
    got = e.device_math("pow_fast", base, expo).astype(np.float64)
    want = base.astype(np.float64) ** expo.astype(np.float64)
    rel_p = (np.abs(got - want) / want - 2.0 ** -22 * np.abs(expo * np.log2(base.astype(np.float64)))).max()
    xs = np.concatenate([rng.uniform(0, 1, 10 ** 6), 10.0 ** rng.uniform(-40, 6, 10 ** 6)]).astype(np.float32)
    got = e.device_math("sqrt_fast", xs).astype(np.float64)
    want = np.sqrt(xs.astype(np.float64))
    rel_q = (np.abs(got - want) / np.where(want > 0, want, 1))[want > 1e-19].max()
    a = (10.0 ** rng.uniform(-30, 30, 10 ** 6)).astype(np.float32)
    b = (10.0 ** rng.uniform(-30, 30, 10 ** 6)).astype(np.float32)
    got = e.device_math("div_fast", a, b).astype(np.float64)
    want = a.astype(np.float64) / b.astype(np.float64)
    fin = (np.abs(want) > 1e-37) & (np.abs(want) < 1e37)
    rel_d = (np.abs(got - want) / np.abs(want))[fin].max()
    print(f"\nfast elementary functions: sin {err_s:.3g} cos {err_c:.3g} (abs), exp {rel_e:.3g}, pow {rel_p:.3g}, sqrt {rel_q:.3g}, "
          f"div {rel_d:.3g} (rel)")
    assert err_s <= Q.SIN_ABS_FAST and err_c <= Q.SIN_ABS_FAST
    assert rel_e <= Q.EXP_REL_FAST and rel_p <= Q.POW_REL_FAST
    assert rel_q <= Q.SQRT_REL_FAST and rel_d <= Q.DIV_REL
    # and they are the approximations, not the strict kernels
    assert (e.device_math("sin_fast", x) != e.device_math("sin", x)).any()
