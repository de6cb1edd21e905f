"""The ReSTIR GI reprojection (K11), temporal resampling (K14), spatial merge (K17) and resolving (K19), pass by pass and value by
value, against the float64 restatement in tests/ref64_restir_gi.py within its derived bound for the arithmetic tier that ran: the
strict oracle on the CPU (with a set of plausible misreadings that the check must catch), and the CUDA kernels of both tiers.

Bit parity with the oracle cannot see a misreading the oracle shares, and the whole-image relative L2 of the fast tier cannot see an
error confined to a few pixels or to the validation frames; these checks see both."""
import numpy as np
import pytest

from strolle_b200 import scenes
from tests import ref64_restir as Q
from tests import ref64_restir_gi as G
from tests.util import Frame, check_within, write_buffer

P_GI_REPROJECTION, P_GI_TEMPORAL, P_GI_SPATIAL_SAMPLE, P_GI_RESOLVING = 7, 10, 13, 15
SEED_BASE = 0xC0FFEE
BRANCHES = ("reprojected", "disoccluded", "confidence reset", "near threshold", "M clamp", "K17 merges", "K17 pass-through",
            "K17 copies", "mutation caught", "normal seam")
# undecided decisions per decision type, as a fraction of the values checked (K17: pairs).  Worst on an H100 over every run of this
# file: `rng W < weight` 1.0e-3 of K17's pairs (normal-mapped room 224x126, fast build) and 2.1e-4 of K14's pixels; K14's `q0 <= 0`
# 8.3e-6 and unbounded pdfs 1.2e-5 (textured room 224x126, fast build).  With the injected edge inputs: `rng W < weight` 2.5e-3
# (K17, strict) and the radiance-distance test 1.0e-3 of K14's pixels (fast build).  No fold or specular decision, and without the
# injected radiances no radiance-distance test, was undecided anywhere.  Caps: twice the worst, and none where none was seen.
UNDECIDED_MAX = {"fold": 0.0, "update": 0.002, "distance": 0.0, "specular": 0.0, "mis q0": 2e-5, "unbounded": 2.5e-5}
UNDECIDED_MAX_EDGES = dict(UNDECIDED_MAX, update=0.005, distance=0.002)
# fraction of the finite nonzero values (K14: m, w and pdf; K19: both outputs) bounded below 1e-3 relative.  Loosest on an H100: the
# normal-mapped room (fast build) with K14 97.7 % and K19 96.7 %: mapped normals put more hits near grazing, where the cosine and the
# specular lobe lose relative precision; Cornell with spot lights 98.1 % for K14 (as for K6, the acos_approx cone term loosens the
# recomputed pdfs, and m takes their ratio to the 8th power).  Strict oracle: K14 98.7 %, K19 99.3 %.
TIGHT_MIN = {"K14": 0.97, "K19": 0.96}


class GiChain:
    """Drives one camera frame by frame on an engine (the CUDA engine or the CPU oracle) and checks K11, K14, K17 and K19 as they
    run, with the inputs of each read just before it and its outputs just after.  `inject`: {pass id: callable(Frame)} run right
    before that pass on every frame.  `rows`: K14 is checked on these rows only."""

    def __init__(self, e, scene, fast, mutation=None, rows=None, expect_caught=()):
        self.e, self.scene, self.fast, self.mutation, self.rows = e, scene, fast, mutation, rows
        self.expect_caught = expect_caught      # K14 mutations that must fail to match the pass's output (counted per frame)
        self.cam = scenes.apply(e, scene)
        c = scene["camera"]
        self.w, self.h = c["w"], c["h"]
        self.t = np.asarray(c["transform"], np.float32).reshape(16).copy()
        self.t_prev = self.t.copy()      # the camera before the last update_camera: the engine's previous camera
        self.stats = {k: [0.0, {}, 0] for k in ("K11", "K14", "K17", "K19")}     # largest ratio, undecided per type, values checked
        self.branches = dict.fromkeys(BRANCHES, 0)
        self.tight = {"K14": [0, 0], "K19": [0, 0]}
        self.f = 0

    def move(self, f):
        c = self.scene["camera"]
        self.t_prev = self.t.copy()
        self.t[12] += np.float32(0.013 * f); self.t[13] += np.float32(0.004 * f)
        self.e.update_camera(self.cam, c["mode"], c["denoise"], c["ref_depth"], self.w, self.h, self.t, c["projection"])

    def _acc(self, key, ratio, und, n):
        s = self.stats[key]
        # decision types differ between frames (the radiance-distance test exists on validation frames only): keep every one seen
        self.stats[key] = [max(s[0], ratio), {k: s[1].get(k, 0) + und.get(k, 0) for k in set(s[1]) | set(und)}, s[2] + n]

    def frame(self, inject=None, checks=(P_GI_REPROJECTION, P_GI_TEMPORAL, P_GI_SPATIAL_SAMPLE, P_GI_RESOLVING)):
        e, cam, w, h, fast, mut = self.e, self.cam, self.w, self.h, self.fast, self.mutation
        inject = inject or {}
        self.f += 1
        f = self.f
        e.tick()
        fr = Frame(e, cam, w, h)
        cur = "b" if f % 2 == 1 else "a"
        old = "a" if cur == "b" else "b"
        proj = self.scene["camera"]["projection"]
        n2w, n2w_prev = Q.ndc_to_world(self.t, proj), Q.ndc_to_world(self.t_prev, proj)
        rd = lambda n: e.read_buffer(cam, n)

        def before(p):
            k = fr.steps(p)
            if not k or p not in checks:
                return None
            fr.run_to(k[0] - 1)
            if p in inject:
                inject[p](fr)
            return k[0]

        k = before(P_GI_REPROJECTION)
        if k is not None:
            d0, d1, rmap, r0, r2 = fr.read(f"prim_gbuffer_d0_{cur}"), fr.read(f"prim_gbuffer_d1_{cur}"), fr.read("reprojection_map"), rd("gi_reservoirs_0"), rd("gi_reservoirs_2")
            r = G.gi_reprojection(n2w, w, h, d0, d1, rmap, r0, fast, mut)
            fr.run_to(k)
            got = rd("gi_reservoirs_2")
            self._acc("K11", G.check_gi(got, r, f"f{f} K11"), r["undecided"], len(r["idx"]))
            self.branches["normal seam"] += r["seam"]
            G.check_untouched(got, r2, r["sky"], f"f{f} K11")
            self.branches["reprojected"] += r["reprojected"]; self.branches["disoccluded"] += r["disoccluded"]
        k = before(P_GI_TEMPORAL)
        if k is not None:
            inline = not fr.steps(P_GI_REPROJECTION)
            gb = [fr.read(f"prim_gbuffer_d{i}_{cur}") for i in (0, 1)]
            gb_prev = [fr.read(f"prim_gbuffer_d{i}_{old}") for i in (0, 1)]
            rmap, r1, r0, r2 = fr.read("reprojection_map"), rd("gi_reservoirs_1"), rd("gi_reservoirs_0"), rd("gi_reservoirs_2")
            r = G.gi_temporal(n2w, n2w_prev, w, h, gb, gb_prev, rmap, r1, r0 if inline else r2,
                              Q.dispatch_seed(SEED_BASE, f, P_GI_TEMPORAL), f, fast, inline, mut, self.rows)
            fr.run_to(k)
            got = rd("gi_reservoirs_1")
            self._acc("K14", G.check_gi(got, r, f"f{f} K14"), r["undecided"], len(r["idx"]))
            self.branches["normal seam"] += r["seam"]
            G.temporal_sky(got, r, f"f{f} K14")
            self.tight["K14"] = [a + b for a, b in zip(self.tight["K14"], G.tight(r, [3, 7, 11]))]
            self.branches["confidence reset"] += r["conf_reset"]; self.branches["M clamp"] += r["m_clamped"]
            self.branches["near threshold"] += r["near_threshold"]
            for m in self.expect_caught:
                # the same inputs through a misread restatement must not match what the pass wrote
                rm = G.gi_temporal(n2w, n2w_prev, w, h, gb, gb_prev, rmap, r1, r0 if inline else r2,
                                   Q.dispatch_seed(SEED_BASE, f, P_GI_TEMPORAL), f, fast, inline, m, self.rows)
                try:
                    G.check_gi(got, rm, f"f{f} K14 {m}")
                except AssertionError:
                    self.branches["mutation caught"] += 1
            if not inline:
                self.branches["reprojected"] += r["reprojected"]; self.branches["disoccluded"] += r["disoccluded"]
            got2 = rd("gi_reservoirs_2")
            if inline:
                # K11 composed in: gi_reservoirs[2] holds K11's reservoir on the columns the checkerboard passes do not cover
                hw = 2 * (8 * (((w + 7) // 8) // 2))
                ys, xs = (a.reshape(-1) for a in np.mgrid[0:h, 0:w])
                tail = xs >= hw
                if self.rows is not None:
                    tail &= np.isin(ys, self.rows)
                r11 = G.gi_reprojection(n2w, w, h, gb[0], gb[1], rmap, r0, fast, mut, xs[tail], ys[tail])
                self._acc("K11", G.check_gi(got2, r11, f"f{f} K11 inline"), r11["undecided"], len(r11["idx"]))
                keep = np.setdiff1d(np.arange(w * h), r11["idx"])
                G.check_untouched(got2, r2, keep, f"f{f} K14 inline (gi_reservoirs_2)")
                self.branches["reprojected"] += r["reprojected"]; self.branches["disoccluded"] += r["disoccluded"]
            else:
                G.check_untouched(got2, r2, np.arange(w * h), f"f{f} K14 (gi_reservoirs_2)")
        k = before(P_GI_SPATIAL_SAMPLE)
        if k is not None:
            r1, r2, d2 = rd("gi_reservoirs_1"), rd("gi_reservoirs_2"), fr.read("gi_d2")
            r = G.gi_spatial_sample(r1, d2, Q.dispatch_seed(SEED_BASE, f, P_GI_SPATIAL_SAMPLE), f, w, h, fast, mut)
            fr.run_to(k)
            got = rd("gi_reservoirs_2")
            ratio = G.check_gi(got, r, f"f{f} K17")
            self.branches["normal seam"] += r["seam"]
            cr, cu = G.check_copies(got, r1, r["copies"], fast, f"f{f} K17 copies")
            und = dict(r["undecided"]); und["fold"] += cu
            self._acc("K17", max(ratio, cr), und, len(r["idx"]))
            G.check_untouched(got, r2, np.setdiff1d(np.arange(w * h), r["written"]), f"f{f} K17")
            self.branches["K17 merges"] += r["merged"]; self.branches["K17 pass-through"] += r["passed"]
            self.branches["K17 copies"] += len(r["copies"])
        k = before(P_GI_RESOLVING)
        if k is not None:
            d0, d1, r0 = fr.read(f"prim_gbuffer_d0_{cur}"), fr.read(f"prim_gbuffer_d1_{cur}"), rd("gi_reservoirs_0")
            src = rd(G.resolving_source(f, mut))
            fr.run_to(k)
            r = G.gi_resolving(n2w, w, h, d0, d1, r0, fast, mut)
            ratio, und = G.check_resolving(fr.read("gi_diff_samples"), fr.read("gi_spec_samples"), r, f"f{f} K19", check_within)
            cr, cu = G.check_copies(rd("gi_reservoirs_0"), src, np.arange(w * h), fast, f"f{f} K19 copy")
            self._acc("K19", max(ratio, cr), {"specular": und, "fold": cu}, int(r["some"].sum()))
            frac, n = Q.tight_fraction([r["diff"], r["spec"]], r["some"])
            self.tight["K19"] = [self.tight["K19"][0] + round(frac * n), self.tight["K19"][1] + n]
        fr.run_to(len(fr.sched) - 1)

    def report(self, tag, limits=None):
        limits = limits or UNDECIDED_MAX
        print(f"\n{tag}: " + "; ".join(f"{k} ratio {s[0]:.3g} undecided {s[1]} of {s[2]}" for k, s in self.stats.items())
              + f"; tight {self.tight}; branches {self.branches}")
        for k, s in self.stats.items():
            for d, v in s[1].items():
                assert v <= limits[d] * max(s[2], 1), f"{tag} {k}: {v} undecided '{d}' of {s[2]}"


def run_chain(e, scene, fast, frames=13, moves=(3, 5, 8, 11), mutation=None, rows=None, inject=None, checks=None, expect_caught=()):
    """The DI tests' schedule: the camera moves on frames 3, 5, 8 and 11; a light is inserted on frame 4, moved on 7 and removed on
    10.  13 frames cover both GI cycles: the validation frames 4, 5, 10 and 11, and moves on validation frames."""
    ch = GiChain(e, scene, fast, mutation, rows, expect_caught)
    for f in range(1, frames + 1):
        if f in moves:
            ch.move(f)
        if f == 4:
            e.insert_light(9001, scenes.LIGHT_POINT, scenes.point_light((0.2, 1.0, 0.3), 0.08, (3.0, 2.0, 1.0), 6.0))
        if f == 7:
            e.insert_light(9001, scenes.LIGHT_POINT, scenes.point_light((-0.3, 0.8, 0.1), 0.08, (3.0, 2.0, 1.0), 6.0))
        if f == 10:
            e.remove_light(9001)
        kw = {} if checks is None else {"checks": checks}
        ch.frame(inject(f) if inject else None, **kw)
    return ch


# ---- CPU: the strict oracle --------------------------------------------------------------------------------------------------

ORACLE_SCENES = {"cornell": lambda: scenes.cornell(64, 40), "demo_level": lambda: scenes.demo_level(64, 36),
                 "cornell_spots": lambda: scenes.cornell_spots(56, 40), "textured_room": lambda: scenes.textured_room(64, 36)}


def _non_vacuous(ch, tag):
    s = ch.stats
    assert all(s[k][2] > 0 for k in s), s
    assert all(1e-3 < s[k][0] <= 1 for k in ("K11", "K14", "K17", "K19")), {k: s[k][0] for k in s}
    for k in ("K14", "K19"):
        t, n = ch.tight[k]
        assert n > 0 and t >= TIGHT_MIN[k] * n, (tag, k, ch.tight[k])
    b = ch.branches
    assert b["reprojected"] > 0 and b["disoccluded"] > 0 and b["K17 merges"] > 0 and b["K17 copies"] > 0, b


@pytest.mark.parametrize("which", sorted(ORACLE_SCENES))
def test_gi_float64_chain_matches_oracle(oracle, blue_noise, which):
    """K11, K14, K17 and K19 of the strict oracle within the float64 restatement's bound, every pixel and pair of 13 frames.  The
    oracle and the CUDA kernels were written from one reading of the reference; this checks that reading against an independent
    one without a GPU."""
    ch = run_chain(oracle.OracleEngine(blue_noise=blue_noise), ORACLE_SCENES[which](), fast=False)
    ch.report(f"oracle {which}")
    _non_vacuous(ch, which)
    assert ch.branches["confidence reset"] > 0 or which == "demo_level", ch.branches


@pytest.mark.parametrize("mutation", G.MUTATIONS)
def test_gi_chain_catches_mutation(oracle, blue_noise, mutation):
    """Each misreading in MUTATIONS, put into the restatement, makes the oracle chain fail on at least one scene."""
    for which in ("cornell", "cornell_spots", "textured_room", "demo_level"):
        try:
            run_chain(oracle.OracleEngine(blue_noise=blue_noise), ORACLE_SCENES[which](), fast=False, mutation=mutation)
        except AssertionError:
            return
    pytest.fail(f"mutation {mutation} passed the oracle chain on every scene")


# ---- GPU -----------------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def gpu():
    import strolle_b200
    return strolle_b200


def _engine(gpu, blue_noise, strict, fused, nmap=False):
    from strolle_b200.engine import OPT_FUSED_PASSES, OPT_NORMAL_MAPS
    e = gpu.Engine(blue_noise=blue_noise, exact=strict)
    e.set_option(OPT_FUSED_PASSES, int(fused))
    e.set_option(OPT_NORMAL_MAPS, int(nmap))
    return e


GPU_SCENES = {"cornell": scenes.cornell, "demo_level": scenes.demo_level, "textured_room": scenes.textured_room,
              "cornell_spots": scenes.cornell_spots, "normal_mapped_room": scenes.normal_mapped_room}
# the fast tier leaves out 67x45: its odd half-grid is covered by the strict tier, and 63x45 covers the off-screen last pair in both
# (this keeps the file near three minutes on one H100)
UNFUSED_CASES = [(s, size, strict) for strict in (True, False) for s in GPU_SCENES
                 for size in (((224, 126), (67, 45), (63, 45)) if strict else ((224, 126), (63, 45)))]


@pytest.mark.gpu
@pytest.mark.parametrize("scene_name,size,strict", UNFUSED_CASES,
                         ids=[f"{s}-{w}x{h}-{'strict' if t else 'fast'}" for s, (w, h), t in UNFUSED_CASES])
def test_gi_unfused_chain_within_float64_bound(gpu, blue_noise, scene_name, size, strict):
    """The unfused schedule, frames 1-13, every pixel and pair: 67x45 (strict) leaves columns K17 never writes (the half grid is 64 wide),
    and on 63x45 the last pair's lhs is off the screen on alternate rows; the normal-mapped room shades with ST_OPT_NORMAL_MAPS."""
    e = _engine(gpu, blue_noise, strict, False, scene_name == "normal_mapped_room")
    ch = run_chain(e, GPU_SCENES[scene_name](*size), fast=not strict)
    ch.report(f"{scene_name} {size} {'strict' if strict else 'fast'}")
    _non_vacuous(ch, scene_name)


PRODUCT_CASES = [(s, size, False) for s in ("cornell", "demo_level", "textured_room") for size in ((224, 126), (63, 45))] + \
                [("cornell", (63, 45), True)]


@pytest.mark.gpu
@pytest.mark.parametrize("scene_name,size,strict", PRODUCT_CASES,
                         ids=[f"{s}-{w}x{h}-{'strict' if t else 'fast'}" for s, (w, h), t in PRODUCT_CASES])
def test_gi_product_default_within_float64_bound(gpu, blue_noise, scene_name, size, strict):
    """The product default (fused passes): K14 with K11 composed in on tracing frames (and gi_reservoirs[2] written only on the
    columns the checkerboard passes do not cover), and the standalone K11 and K14 it still runs on validation frames."""
    e = _engine(gpu, blue_noise, strict, True)
    ch = run_chain(e, GPU_SCENES[scene_name](*size), fast=not strict)
    assert ch.stats["K17"][2] == 0 and ch.stats["K19"][2] == 0 and ch.stats["K14"][2] > 0 and ch.stats["K11"][2] > 0
    assert 1e-3 < ch.stats["K14"][0] <= 1 and ch.branches["reprojected"] > 0
    ch.report(f"{scene_name} {size} product default{' (strict)' if strict else ''}")


@pytest.mark.gpu
def test_gi_1080p_product_default(gpu, blue_noise):
    """Frames 1-5 of the product default at 1920x1080; K14 on a band of 32 rows on frames 2, 4 and 5 (a gathering frame, a
    validation frame with K11 standalone, and one more)."""
    e = _engine(gpu, blue_noise, False, True)
    ch = GiChain(e, scenes.cornell(1920, 1080), fast=True, rows=np.arange(524, 556))
    for f in range(1, 6):
        ch.frame(checks=(P_GI_TEMPORAL,) if f in (2, 4, 5) else ())
    assert ch.stats["K14"][2] > 0 and 1e-3 < ch.stats["K14"][0] <= 1
    ch.report("1080p product default")


# ---- injected edge inputs ------------------------------------------------------------------------------------------------------

def _reservoir_edges(name, seed, m=True, w=True, pdf=True, v2=True):
    """Rewrites a GI reservoir buffer: M at 127, 128, 129 and 1e6, w at 0, a denormal, 5 and 1e6, pdf 0, v2 (0, 0, 0) and
    (-0, 0, 0), on live reservoirs picked at random."""
    def inject(fr):
        rng = np.random.RandomState(seed)
        r = fr.e.read_buffer(fr.cam, name).reshape(-1, 16).copy()
        live = r[:, 3] > 0
        k = rng.randint(0, 14, len(r))
        pick = lambda j: live & (k == j)
        if m:
            for j, v in ((1, 127), (2, 128), (3, 129), (4, 1e6)):
                r[pick(j), 3] = v
        if w:
            for j, v in ((5, 0), (6, np.float32(1e-41)), (7, 5), (8, 1e6)):
                r[pick(j), 7] = v
        if pdf:
            r[pick(9), 11] = 0
        if v2:
            r[pick(10), 8:11] = 0
            r[pick(11), 8:11] = np.array([-0.0, 0.0, 0.0], np.float32)
        write_buffer(fr.e, fr.cam, name, r.astype(np.float32))
    return inject


def _radiance_near_threshold(seed):
    """On a validation frame, before K14: the current reservoirs' radiance set to the reprojected one's plus a vector of length
    0.33 +- a few ulp (and exactly 0.33), so the radiance-distance test meets its threshold."""
    def inject(fr):
        rng = np.random.RandomState(seed)
        r1 = fr.e.read_buffer(fr.cam, "gi_reservoirs_1").reshape(-1, 16).copy()
        r2 = fr.e.read_buffer(fr.cam, "gi_reservoirs_2").reshape(-1, 16)
        sel = (r1[:, 3] > 0) & (r2[:, 3] > 0) & (rng.rand(len(r1)) < 0.3)
        d = np.float32(0.33) + (rng.randint(-4, 5, len(r1)) * np.spacing(np.float32(0.33))).astype(np.float32)
        ax = rng.randint(0, 3, len(r1))
        for a in range(3):
            s = sel & (ax == a)
            r1[s, a] = r2[s, a] + d[s]
        write_buffer(fr.e, fr.cam, "gi_reservoirs_1", r1.astype(np.float32))
    return inject


def _texel_edges(seed):
    """Before K17: some pairs' texel a gets rhs_idx + 1 of 0, w h + 1 or 0xFFFFFFFF.  K17 (gi_spatial_sample_pair) merges only where
    rhs_idx > 0 and rhs_idx - 1 < w h, so the last two read nothing: it passes the lhs through."""
    def inject(fr):
        rng = np.random.RandomState(seed)
        d2 = fr.read("gi_d2").copy()
        bits = d2[..., 1].view(np.uint32).copy()
        k = rng.randint(0, 6, bits.shape)
        even = (np.arange(fr.w) % 2 == 0)[None, :]       # texel a of each pair
        bits = np.where(even & (k == 1), 0, np.where(even & (k == 2), fr.w * fr.h + 1, np.where(even & (k == 3), 0xFFFFFFFF, bits)))
        d2[..., 1] = bits.astype(np.uint32).view(np.float32)
        fr.write("gi_d2", d2)
    return inject


def _gbuffer_edges(seed, cur_of):
    """Before K19: metallic and roughness bytes at 0 and 255 on random surface pixels."""
    def inject(fr):
        rng = np.random.RandomState(seed)
        name = f"prim_gbuffer_d0_{cur_of()}"
        d0 = fr.read(name).copy()
        bits = d0[..., 3].view(np.uint32).copy()
        mb, rb = bits & 0xFF, (bits >> 8) & 0xFF
        k = rng.randint(0, 5, bits.shape)
        mb = np.where(k == 1, 0, np.where(k == 2, 255, mb)); rb = np.where(k == 3, 0, np.where(k == 4, 255, rb))
        d0[..., 3] = ((bits & 0xFFFF0000) | mb | (rb << 8)).astype(np.uint32).view(np.float32)
        fr.write(name, d0)
    return inject


@pytest.mark.gpu
@pytest.mark.parametrize("strict", [True, False], ids=["strict", "fast"])
def test_gi_edge_inputs_within_bound(gpu, blue_noise, strict):
    """Edge contents written just before the pass that reads them, on the textured room at 67x45 over 13
    frames: K11's source (gi_reservoirs[0]) and K14's reprojected reservoirs (gi_reservoirs[2]) with M at the clamp of 128 and far
    past it, w at 0, a denormal, 5 and 1e6, pdf 0 and v2 of +-0 (K14 restated with M clamped at 64 must not match there); on
    validation frames radiances 0.33 +- a few ulp apart; K17's
    reservoirs likewise and its texels with rhs_idx + 1 of 0, w h + 1 and 0xFFFFFFFF; K19's G-buffer bytes at 0 and 255."""
    e = _engine(gpu, blue_noise, strict, False)
    scene = scenes.textured_room(67, 45)
    holder = {}

    def inject(f):
        holder["cur"] = "b" if f % 2 == 1 else "a"
        k14 = [_reservoir_edges("gi_reservoirs_2", 10 * f)]
        if not G.tracing_frame(f):
            k14.append(_radiance_near_threshold(10 * f + 1))
        return {P_GI_REPROJECTION: _reservoir_edges("gi_reservoirs_0", 10 * f + 2),
                P_GI_TEMPORAL: lambda fr: [g(fr) for g in k14],
                P_GI_SPATIAL_SAMPLE: lambda fr: (_reservoir_edges("gi_reservoirs_1", 10 * f + 3, v2=False)(fr), _texel_edges(10 * f + 4)(fr)),
                P_GI_RESOLVING: lambda fr: (_reservoir_edges("gi_reservoirs_0", 10 * f + 5, m=False, pdf=False)(fr),
                                            _gbuffer_edges(10 * f + 6, lambda: holder["cur"])(fr))}
    ch = run_chain(e, scene, fast=not strict, inject=inject, expect_caught=("k14_m64",))
    ch.report(f"edges {'strict' if strict else 'fast'}", UNDECIDED_MAX_EDGES)
    assert ch.branches["M clamp"] > 0 and ch.branches["confidence reset"] > 0 and ch.branches["K17 pass-through"] > 0, ch.branches
    # the injected radiances reach the 0.33 threshold (within 1e-5 of it, decided or not), and K14 restated with M clamped at 64
    # instead of 128 fails to match the pass on some frame
    assert ch.branches["near threshold"] > 0 and ch.branches["mutation caught"] > 0, ch.branches
    assert all(ch.stats[k][2] > 0 for k in ch.stats), ch.stats


@pytest.mark.gpu
def test_gi_fast_shading_build_is_not_strict(gpu, blue_noise):
    """The fast-tier runs really ran the fast build: K14 and K19 rerun with the strict build on the same inputs give different bits
    somewhere."""
    from strolle_b200.engine import OPT_SHADING_FAST_MATH
    e = _engine(gpu, blue_noise, False, False)
    cam = scenes.apply(e, scenes.textured_room(67, 45))
    e.tick(); e.render_camera(cam)
    e.tick()     # frame 2: a gathering frame (K12 / K13 sample, K14 resamples)
    fr = Frame(e, cam, 67, 45)
    k14, k19 = fr.steps(P_GI_TEMPORAL)[0], fr.steps(P_GI_RESOLVING)[0]
    fr.run_to(k14 - 1)
    pre = e.read_buffer(cam, "gi_reservoirs_1").copy()
    fr.run_to(k14)
    fast14 = e.read_buffer(cam, "gi_reservoirs_1").copy()
    fr.run_to(k19 - 1)
    pre0 = e.read_buffer(cam, "gi_reservoirs_0").copy()
    fr.run_to(k19)
    fast19 = fr.read("gi_diff_samples").copy(), fr.read("gi_spec_samples").copy()
    e.set_option(OPT_SHADING_FAST_MATH, 0)
    write_buffer(e, cam, "gi_reservoirs_0", pre0)
    e.render_range(cam, k19, k19)
    strict19 = fr.read("gi_diff_samples"), fr.read("gi_spec_samples")
    assert any((a.view(np.uint32) != b.view(np.uint32)).any() for a, b in zip(fast19, strict19)), "K19"
    write_buffer(e, cam, "gi_reservoirs_1", pre)
    e.render_range(cam, k14, k14)
    assert (e.read_buffer(cam, "gi_reservoirs_1").view(np.uint32) != fast14.view(np.uint32)).any(), "K14"


# ---- the sky ---------------------------------------------------------------------------------------------------------------------

P_DI_RESOLVING = 6
SKY_SUN_AZIMUTH = 3.0
# the demo level's sun, the sun below the horizon of Cornell and the normal-mapped room, and a low sun whose bloom crosses the horizon
# (where the ground test decides whether the sun adds to the sky)
SKY_SUN_ALTITUDES = (0.35, -1.0, 0.05)


def _look(dir_, fov, up=(0.0, 1.0, 0.0)):
    return dict(transform=scenes.look_at_transform((0.0, 0.0, 0.0), dir_, up), projection=scenes.perspective_infinite_reverse_rh(fov, 1.5, 0.1))


def _sun_vec(alt):
    return (np.cos(alt) * np.sin(SKY_SUN_AZIMUTH), np.sin(alt), -np.cos(alt) * np.cos(SKY_SUN_AZIMUTH))


def sky_views(alt):
    """Camera views of the sky scene with the sun at altitude `alt`: the sun disc (narrow) and its bloom, the nadir (where
    sample_sky_lut's |altitude| > pi / 2 - 1e-4 branch is taken) and the zenith, the horizon and below it, and the direction opposite
    the sun, across which u jumps between 0 and 1."""
    sun = np.array(_sun_vec(alt))
    anti = np.array(_sun_vec(0.15)) * np.array([-1.0, 1.0, -1.0])
    side = np.array(_sun_vec(0.0))[[2, 1, 0]] * np.array([1.0, 1.0, -1.0])
    return [_look(sun, 0.05), _look(sun, 0.5), _look((0.0, -1.0, 0.0), 0.05, (0.0, 0.0, 1.0)), _look((0.0, 1.0, 0.0), 0.3, (0.0, 0.0, 1.0)),
            _look(side, 0.3), _look(side + np.array([0.0, -0.4, 0.0]), 0.3), _look(anti, 0.3)]


def sky_scene(w=48, h=32):
    """No geometry in view: one small triangle far below and to the side (the engine builds a BVH of it), the sun at azimuth 3.0."""
    tri = scenes.tri36([[-2000.0, -3000.0, 0.0], [-2000.0, -3000.0, 1.0], [-2001.0, -3000.0, 0.0]], [[0.0, 1.0, 0.0]] * 3)
    v = sky_views(0.35)[0]
    cam = dict(mode=scenes.MODE_IMAGE, denoise=True, ref_depth=1, w=w, h=h, **v)
    return dict(name="sky", meshes={1: tri[None]}, materials={1: (scenes.material((0.5, 0.5, 0.5, 1.0)), False)},
                instances=[(1, 1, 1, scenes.IDENTITY_AFFINE)], lights=[], sun=(SKY_SUN_AZIMUTH, 0.35), camera=cam)


# undecided sky decisions, as a fraction of the sky pixels checked.  Worst on an H100 (fast build, 32220 pixels): the sun disc 2.7e-3,
# the nadir branch 1.1e-3, an acos argument that may round past -1 (not compared) 1.1e-3; the strict build and the oracle 7.4e-4,
# 1.1e-3 and 3.7e-4.  No atan2 cut or ground test was undecided.  Caps: about twice the worst, and none where none was seen.
# Fraction of the finite nonzero sky values bounded below 1e-3 relative: 66.9 % in the fast build, 72.5 % strict.  The sun's bloom
# multiplies cos theta's rounding by 50000 and sqrt(|altitude|) near the horizon by its unbounded slope, so the views aimed there
# are loosely bounded by nature.
SKY_UNDECIDED_MAX = {"nadir": 0.0025, "atan2 cut": 0.0, "sun disc": 0.006, "ground": 0.0, "acos domain": 0.0025}
SKY_TIGHT_MIN = 0.6


def run_sky(e, fast, mutation=None):
    """Every view of sky_views at each of SKY_SUN_ALTITUDES: K10's sky pixels (every pixel of these views) against
    Atmosphere::sample.  Returns (largest ratio, undecided per decision, pixels, branches, [tight, finite nonzero])."""
    scene = sky_scene()
    c = scene["camera"]
    w, h = c["w"], c["h"]
    cam = scenes.apply(e, scene)
    ratio, und, npx, tight = 0.0, {}, 0, [0, 0]
    branches = dict.fromkeys(Q.SKY_BRANCHES, 0)
    f = 0
    for alt in SKY_SUN_ALTITUDES:
        e.update_sun(SKY_SUN_AZIMUTH, alt)
        for v in sky_views(alt):
            e.update_camera(cam, c["mode"], c["denoise"], c["ref_depth"], w, h, v["transform"], v["projection"])
            e.tick()
            f += 1
            fr = Frame(e, cam, w, h)
            k10 = fr.steps(P_DI_RESOLVING)[0]
            fr.run_to(k10 - 1)
            d0, d1, r2 = fr.read("prim_gbuffer_d0_b" if f % 2 else "prim_gbuffer_d0_a"), fr.read("prim_gbuffer_d1_b" if f % 2 else "prim_gbuffer_d1_a"), e.read_buffer(cam, "di_reservoirs_2")
            fr.run_to(k10)
            assert (d0[..., 0] == 0).all(), "the sky scene's views must see no geometry"
            r = Q.di_resolving(Q.ndc_to_world(v["transform"], v["projection"]), w, h, d0, d1, e.read_scene("lights"), r2,
                               e.read_buffer(cam, "di_reservoirs_0"), fast, Q.atmosphere_inputs(e), mutation)
            ratio = max(ratio, Q.check_resolving(fr.read("di_diff_samples"), fr.read("di_spec_samples"), e.read_buffer(cam, "di_reservoirs_0"),
                                                 r, f"sky alt {alt} view {f}", check_within)[0])
            s = r["sky"]
            for k, m in s["undecided"].items():
                und[k] = und.get(k, 0) + int(m.sum())
            for k, n in s["branches"].items():
                branches[k] += n
            npx += int(s["domain"].sum())
            frac, n = Q.tight_fraction([s["diff"]], s["domain"])
            tight = [tight[0] + round(frac * n), tight[1] + n]
            fr.run_to(len(fr.sched) - 1)
    return ratio, und, npx, branches, tight


def _sky_ok(res, tag):
    ratio, und, npx, branches, tight = res
    print(f"\n{tag}: sky ratio {ratio:.3g}, undecided {und} of {npx}, branches {branches}, tight {tight}")
    assert npx > 0 and 1e-3 < ratio <= 1, (npx, ratio)
    assert all(v > 0 for v in branches.values()), branches
    assert all(v <= SKY_UNDECIDED_MAX[k] * npx for k, v in und.items()), und
    assert tight[0] >= SKY_TIGHT_MIN * tight[1], tight


def test_sky_oracle_within_float64_bound(oracle, blue_noise):
    """K10's sky pixels of the strict oracle against Atmosphere::sample in float64, over the sky scene's views."""
    _sky_ok(run_sky(oracle.OracleEngine(blue_noise=blue_noise), False), "oracle sky")


@pytest.mark.parametrize("mutation", Q.SKY_MUTATIONS)
def test_sky_catches_mutation(oracle, blue_noise, mutation):
    """Each misreading of atmosphere.rs in SKY_MUTATIONS, put into the restatement, fails the sky check on the oracle."""
    with pytest.raises(AssertionError):
        run_sky(oracle.OracleEngine(blue_noise=blue_noise), False, mutation)


@pytest.mark.gpu
@pytest.mark.parametrize("strict", [True, False], ids=["strict", "fast"])
def test_sky_within_float64_bound(gpu, blue_noise, strict):
    """K10's sky pixels on the device, both tiers, over the sky scene's views."""
    _sky_ok(run_sky(_engine(gpu, blue_noise, strict, False), not strict), f"sky {'strict' if strict else 'fast'}")
