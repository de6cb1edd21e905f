"""The DI sampling (K5), temporal resampling (K6), spatial merge (K9) and resolving (K10) on the device, pass by pass and value by value, against the
float64 restatement in
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

P_DI_SAMPLING, P_DI_TEMPORAL, P_DI_SPATIAL_PICK, P_DI_SPATIAL_TRACE, P_DI_SPATIAL_SAMPLE, P_DI_RESOLVING = 1, 2, 3, 4, 5, 6
SCRATCH = ("di_diff_samples", "di_diff_curr_colors", "di_diff_stash")
SEED_BASE = 0xC0FFEE
SCENES = {"cornell": scenes.cornell, "demo_level": scenes.demo_level, "textured_room": scenes.textured_room,
          "cornell_spots": lambda w, h: scenes.cornell_spots(w, h), "cornell_many_lights": scenes.cornell, "cornell_remap": scenes.cornell,
          "normal_mapped_room": scenes.normal_mapped_room}
# undecided decisions allowed per pass, as a fraction of the values checked.  None were seen in the scene runs on an H100 (24 runs, both
# tiers); the injected M = 1e6 / w = 1e6 reservoirs put 3.6 % of K9's merges inside the bound of `rng W < weight` (W dominated by the
# huge weight, the other weight below its rounding), hence the looser limit there.
UNDECIDED_MAX = 0.001
UNDECIDED_MAX_EDGES = 0.1
# K8's visibility bit against trace_any of the ray decoded in strict f32, as a fraction of the rays traced.  The strict build must
# agree on every ray; the fast build decodes the octahedral direction with FMA contraction, so a ray grazing an edge may differ.
# Worst seen in the fast scene runs on an H100: 3 of 29164 rays (1.0e-4, textured room 67x45); the cap is 1e-3 of the rays traced.
# The fused K7-K9 launch, against the rays of K7's restatement rebuilt in strict f32: 55 of 238198 rays (2.3e-4, textured room
# 224x126, fast build), 0 in the strict build.
K8_DISAGREE_MAX = 1e-3
K5_EVERY_FRAME_PX = 67 * 45     # screens up to this size check K5 on every frame, larger ones on every third (Chain.frame)
# K7 pairs with an undecided decision (a tap coordinate within its bound of an integer, a depth or normal test or `pdf > 0` within
# its bound, an octahedral fold sign), as a fraction of the pairs checked, for K7 alone and for the fused K7-K9 launch (plus K9's
# undecided merges there).  Worst seen on an H100 (every run of this file, both tiers): 1.3e-3 (fused K7-K9, textured room 67x45, fast
# build, with empty reservoirs injected); K7 alone 9.1e-4.  The cap is 1.5 times the worst.
K7_UNDECIDED_MAX = 0.002
# The fused K5 + K6 launch against K5 composed into K6, per decision type, as a fraction of the pixels checked.  K6's lhs light point
# now carries K5's bound, and Light::ray_bnoise puts it near the light's sphere, so `Light::contains` (|center - point| <= radius) is
# often decided inside that bound.  Worst seen on an H100 (fast build): contains 5.4e-3 (textured room 224x126), K6's updates 2.3e-3
# (Cornell with spot lights, 67x45), K5's selection or sign 7.4e-4; the cap is about twice the worst.
FUSED_K6_UNDECIDED_MAX = 0.01


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


class Chain:
    """Drives one camera frame by frame and checks K5, K6, K7, K8, K9 (these five in the unfused schedule), the fused K7 + K8 + K9
    launch against K7, K8 and K9 composed, and K10 as they run.  `rows`: the fused launch is checked on these rows only."""

    def __init__(self, gpu, blue_noise, scene, strict, fused, nmap=False, rows=None):
        self.e = _engine(gpu, blue_noise, strict, fused, nmap)
        self.rows = rows
        self.scene = scene
        self.cam = scenes.apply(self.e, scene)
        c = scene["camera"]
        self.w, self.h = c["w"], c["h"]
        self.t = np.asarray(c["transform"], np.float32).reshape(16).copy()
        self.t_prev = self.t.copy()     # the camera before the last update_camera: the engine's previous camera
        self.fast = not strict
        self.blue_noise = blue_noise
        self.stats = {"K9": [0.0, 0, 0], "K10": [0.0, 0, 0], "K6": [0.0, {}, 0], "K8": [0, 0], "K5": [0.0, {}, 0, 0, 0],
                      "K7": [0.0, 0, 0], "K7-K9": [0.0, 0, 0, 0, 0],   # K7-K9: K9 ratio, undecided, merges, rays, disagreements
                      "K5-K6": [0.0, {}, 0, 0]}    # ratio, undecided per decision type, pixels (one shadow ray each), disagreements
        self.k7_tight = [0, 0]
        self.k7_branches = dict.fromkeys(Q.K7_BRANCHES, 0)
        self.k5_tight = {k: [0, 0] for k in ("w", "light_point")}
        self.k6_tight = {k: [0, 0] for k in ("m", "w", "pdf")}
        self.k6_branches = [0, 0, 0]    # reprojected, killed, remapped
        self.k9_tight = [0, 0]     # (tightly bounded, finite nonzero) m and w of the merged pairs
        self.bounds = []
        self.f = 0

    def move(self, f):
        c = self.scene["camera"]
        self.t_prev = self.t.copy()
        self.t[12] += np.float32(0.013 * f); self.t[13] += np.float32(0.004 * f)
        self.e.update_camera(self.cam, c["mode"], c["denoise"], c["ref_depth"], self.w, self.h, self.t, c["projection"])

    def _check_sampling(self, fr, cur):
        e, cam, w, h, f = self.e, self.cam, self.w, self.h, self.f
        k5 = fr.steps(P_DI_SAMPLING)[0]
        fr.run_to(k5 - 1)
        r1 = e.read_buffer(cam, "di_reservoirs_1")
        r = Q.di_sampling(Q.ndc_to_world(self.t, self.scene["camera"]["projection"]), w, h, fr.read(f"prim_gbuffer_d0_{cur}"),
                          fr.read(f"prim_gbuffer_d1_{cur}"), e.read_scene("lights"), e.read_scene("world")[:1].view(np.uint32)[0],
                          self.blue_noise, Q.dispatch_seed(SEED_BASE, f, P_DI_SAMPLING), f, self.fast)
        fr.run_to(k5)
        s5 = Q.check_sampling(e.read_buffer(cam, "di_reservoirs_1"), r1, r, lambda x: e.device_math("sin", x),
                              lambda x: e.device_math("cos", x), e.trace_any, f"f{f} K5")
        if not self.fast:
            assert s5["disagree"] == 0, f"f{f} K5: {s5['disagree']} of {s5['traced']} occluded bits differ from trace_any"
            lp = s5["got"][:, 4:7]
            assert (lp.view(np.uint32) == s5["lp_f32"].view(np.uint32)).all(), f"f{f} K5: light point differs from its strict f32 rebuild"
        s = self.stats["K5"]
        self.stats["K5"] = [max(s[0], s5["ratio"]), {k: s[1].get(k, 0) + v for k, v in s5["undecided"].items()}, s[2] + s5["n"],
                            s[3] + s5["traced"], s[4] + s5["disagree"]]
        for k, (tt, nn) in s5["tight"].items():
            self.k5_tight[k][0] += tt; self.k5_tight[k][1] += nn

    def _pick(self, fr, cur, inject_k7, rows=None):
        """Runs to the launch before K7 (or the fused K7 + K8 + K9), injects, and restates K7 on what the launch will read: returns
        (restatement, di_reservoirs[1], the three scratch buffers as they were)."""
        e, f = self.e, self.f
        k7 = fr.steps(P_DI_SPATIAL_PICK)[0]
        fr.run_to(k7 - 1)
        if inject_k7:
            inject_k7(fr)
        r1 = e.read_buffer(self.cam, "di_reservoirs_1")
        scratch = [fr.read(n).copy() for n in SCRATCH]
        r = Q.di_spatial_pick(Q.ndc_to_world(self.t, self.scene["camera"]["projection"]), self.w, self.h, fr.read(f"prim_gbuffer_d0_{cur}"),
                              fr.read(f"prim_gbuffer_d1_{cur}"), e.read_scene("lights"), r1, Q.dispatch_seed(SEED_BASE, f, P_DI_SPATIAL_PICK),
                              f, self.fast, rows)
        self.k7_branches = {k: self.k7_branches[k] + v for k, v in r["branches"].items()}
        fr.run_to(k7)
        return r, r1, scratch

    def _check_fused_spatial(self, fr, cur, inject_k7):
        """k_di_spatial_fused against K7, K8 (trace_any of each ray rebuilt in strict f32) and K9 composed, on self.rows.  The strict
        build must agree with every rebuilt ray; in the fast build a pair matched only with a flipped visibility bit counts as a
        disagreement.  The scratch textures are left as they were."""
        e, f = self.e, self.f
        r7, r1, scratch = self._pick(fr, cur, inject_k7, self.rows)
        for n, a in zip(SCRATCH, scratch):
            assert (fr.read(n).view(np.uint32) == a.view(np.uint32)).all(), f"f{f} fused K7-K9 wrote {n}"
        st = Q.pick_stash(r7, e.trace_any)
        seed = Q.dispatch_seed(SEED_BASE, f, P_DI_SPATIAL_SAMPLE)
        flips = [(False, False)] if not self.fast else [(False, False), (True, False), (False, True), (True, True)]
        r = Q.merge_alternatives([Q.di_spatial_sample(r1, Q.flip_visibility(st, a, b), seed, f, self.w, self.h, self.fast, self.rows, a + b)
                                  for a, b in flips])
        ratio, und, merged, flipped = Q.check_spatial_sample(e.read_buffer(self.cam, "di_reservoirs_2"), r1, r, f"f{f} fused K7-K9")
        s = self.stats["K7-K9"]
        self.stats["K7-K9"] = [max(s[0], ratio), s[1] + und + int(r7["undecided"].sum()), s[2] + merged,
                               s[3] + int(st["traced_a"].sum() + st["traced_b"].sum()), s[4] + flipped]

    def _check_fused_temporal(self, fr, cur, old, restate):
        """k_di_sample_temporal against K5 composed into K6 (sampling_lhs into di_temporal), inputs read just before the launch.  The
        strict build must agree with trace_any of every shadow ray rebuilt in strict f32; in the fast build a pixel matched only with
        its occluded bit flipped counts as a disagreement.  Without `restate` only the scratch textures are checked (left alone)."""
        e, cam, w, h, f = self.e, self.cam, self.w, self.h, self.f
        kt = fr.steps(P_DI_TEMPORAL)[0]
        fr.run_to(kt - 1)
        scratch = [fr.read(n).copy() for n in SCRATCH]
        if restate:
            proj = self.scene["camera"]["projection"]
            n2w = Q.ndc_to_world(self.t, proj)
            gb = [fr.read(f"prim_gbuffer_d{k}_{cur}") for k in (0, 1)]
            gb_prev = [fr.read(f"prim_gbuffer_d{k}_{old}") for k in (0, 1)]
            r1, r0, lights = e.read_buffer(cam, "di_reservoirs_1"), e.read_buffer(cam, "di_reservoirs_0"), e.read_scene("lights")
            k5 = Q.di_sampling(n2w, w, h, gb[0], gb[1], lights, e.read_scene("world")[:1].view(np.uint32)[0], self.blue_noise,
                               Q.dispatch_seed(SEED_BASE, f, P_DI_SAMPLING), f, self.fast)
            lhs = Q.sampling_lhs(k5, lambda x: e.device_math("sin", x), lambda x: e.device_math("cos", x), e.trace_any)
            args = (n2w, Q.ndc_to_world(self.t_prev, proj), w, h, gb, gb_prev, fr.read("reprojection_map"), lights, None, r0,
                    Q.dispatch_seed(SEED_BASE, f, P_DI_TEMPORAL), self.fast)
            rs = [Q.di_temporal(*args, lhs=lhs)]
            if self.fast:
                rs.append(Q.di_temporal(*args, lhs=dict(lhs, occ=~lhs["occ"]), flips=1))
            r = Q.merge_temporal(rs)
        fr.run_to(kt)
        for n, a in zip(SCRATCH, scratch):
            assert (fr.read(n).view(np.uint32) == a.view(np.uint32)).all(), f"f{f} fused K5-K6 wrote {n}"
        if restate:
            ratio, und, n, flipped = Q.check_temporal(e.read_buffer(cam, "di_reservoirs_1"), r1, r, f"f{f} fused K5-K6")
            s = self.stats["K5-K6"]
            self.stats["K5-K6"] = [max(s[0], ratio), {k: s[1].get(k, 0) + v for k, v in und.items()}, s[2] + n, s[3] + flipped]

    def _k7_stats(self, s7):
        s = self.stats["K7"]
        self.stats["K7"] = [max(s[0], s7["ratio"]), s[1] + s7["undecided"], s[2] + s7["pairs"]]
        self.k7_tight = [a + b for a, b in zip(self.k7_tight, s7["tight"])]

    def frame(self, inject_k9=None, inject_k10=None, inject_k6=None, inject_k7=None):
        e, cam, w, h = self.e, self.cam, self.w, self.h
        self.f += 1
        f = self.f
        e.tick()
        fr = Frame(e, cam, w, h)
        cur = "b" if f % 2 == 1 else "a"
        old = "a" if cur == "b" else "b"
        k9 = fr.steps(P_DI_SPATIAL_SAMPLE)
        if not k9:   # fused schedule: k_di_sample_temporal (pass 2), then k_di_spatial_fused (pass 3)
            # as for K5 in the unfused schedule, screens above K5_EVERY_FRAME_PX check pass 2 on every third frame
            self._check_fused_temporal(fr, cur, old, self.rows is None and (w * h <= K5_EVERY_FRAME_PX or f % 3 == 1))
            self._check_fused_spatial(fr, cur, inject_k7)
        if k9:   # unfused schedule: K5 writes its samples to di_reservoirs[1], K6 reads them from there
            # K5 carries no state from frame to frame, so above K5_EVERY_FRAME_PX pixels it is checked on every third frame (1, 4, 7,
            # 10, 13: the frames that insert, move and remove a light); its f64 restatement is the costliest of the chain
            if w * h <= K5_EVERY_FRAME_PX or f % 3 == 1:
                self._check_sampling(fr, cur)
            k6 = fr.steps(P_DI_TEMPORAL)[0]
            fr.run_to(k6 - 1)
            if inject_k6:
                inject_k6(fr)
            gb = [fr.read(f"prim_gbuffer_d{k}_{cur}") for k in (0, 1)]
            gb_prev = [fr.read(f"prim_gbuffer_d{k}_{old}") for k in (0, 1)]
            r1, r0 = e.read_buffer(cam, "di_reservoirs_1"), e.read_buffer(cam, "di_reservoirs_0")
            proj = self.scene["camera"]["projection"]
            r = Q.di_temporal(Q.ndc_to_world(self.t, proj), Q.ndc_to_world(self.t_prev, proj), w, h, gb, gb_prev, fr.read("reprojection_map"),
                              e.read_scene("lights"), r1, r0, Q.dispatch_seed(SEED_BASE, f, P_DI_TEMPORAL), self.fast)
            fr.run_to(k6)
            ratio, und, n, _ = Q.check_temporal(e.read_buffer(cam, "di_reservoirs_1"), r1, r, f"f{f} K6")
            s = self.stats["K6"]
            self.stats["K6"] = [max(s[0], ratio), {k: s[1].get(k, 0) + v for k, v in und.items()}, s[2] + n]
            for k, (tt, nn) in Q.temporal_tight(r).items():
                self.k6_tight[k][0] += tt; self.k6_tight[k][1] += nn
            self.k6_branches = [a + r[b] for a, b in zip(self.k6_branches, ("reprojected", "killed", "remapped"))]
            # K7 too carries no state from frame to frame: above K5_EVERY_FRAME_PX pixels it is checked on K5's frames
            if w * h <= K5_EVERY_FRAME_PX or f % 3 == 1:
                r7, _, (p0, p1, _) = self._pick(fr, cur, inject_k7)
                self._k7_stats(Q.check_spatial_pick(fr.read("di_diff_samples"), fr.read("di_diff_curr_colors"), p0, p1, r7, f"f{f} K7"))
            k8 = fr.steps(P_DI_SPATIAL_TRACE)[0]
            fr.run_to(k8 - 1)
            b0, b1 = fr.read("di_diff_samples"), fr.read("di_diff_curr_colors")
            fr.run_to(k8)
            traced, bad = Q.check_spatial_trace(b0, b1, fr.read("di_diff_stash"), e.trace_any, f"f{f} K8")
            if not self.fast:
                assert bad == 0, f"f{f} K8: {bad} of {traced} visibility bits differ from trace_any"
            self.stats["K8"] = [self.stats["K8"][0] + traced, self.stats["K8"][1] + bad]
        if k9:   # unfused schedule: K9 reads K8's visibility texels from di_diff_stash
            fr.run_to(k9[0] - 1)
            if inject_k9:
                inject_k9(fr)
            r1, stash = e.read_buffer(cam, "di_reservoirs_1"), fr.read("di_diff_stash")
            fr.run_to(k9[0])
            r = Q.di_spatial_sample(r1, stash, Q.dispatch_seed(SEED_BASE, f, P_DI_SPATIAL_SAMPLE), f, w, h, self.fast)
            ratio, und, merged, _ = Q.check_spatial_sample(e.read_buffer(cam, "di_reservoirs_2"), r1, r, f"f{f} K9")
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
        r = Q.di_resolving(Q.ndc_to_world(self.t, self.scene["camera"]["projection"]), w, h, d0, d1, e.read_scene("lights"), r2, res0, self.fast,
                            Q.atmosphere_inputs(e))
        ratio, und, b = Q.check_resolving(fr.read("di_diff_samples"), fr.read("di_spec_samples"), res0, r, f"f{f} K10", check_within)
        s = self.stats["K10"]
        self.stats["K10"] = [max(s[0], ratio), s[1] + und, s[2] + int(r["some"].sum())]
        self.bounds.append((b, r["some"]))
        fr.run_to(len(fr.sched) - 1)
        return r

    def report(self, tag, limit=UNDECIDED_MAX):
        s9, s10, s6, s8, s5 = self.stats["K9"], self.stats["K10"], self.stats["K6"], self.stats["K8"], self.stats["K5"]
        s7, sf, st = self.stats["K7"], self.stats["K7-K9"], self.stats["K5-K6"]
        print(f"\n{tag}: K5 ratio {s5[0]:.3g} undecided {s5[1]} of {s5[2]}, shadow rays differ {s5[4]}/{s5[3]}, tight {self.k5_tight}; "
              f"K6 ratio {s6[0]:.3g} undecided {s6[1]} of {s6[2]}, reprojected / killed / remapped {self.k6_branches}; "
              f"K8 visibility differs {s8[1]}/{s8[0]}; K9 ratio {s9[0]:.3g} undecided {s9[1]}/{s9[2]}; "
              f"K10 ratio {s10[0]:.3g} undecided specular {s10[1]}/{s10[2]}; "
              f"K7 ratio {s7[0]:.3g} undecided {s7[1]}/{s7[2]} tight {self.k7_tight} branches {self.k7_branches}; "
              f"fused K7-K9 ratio {sf[0]:.3g} undecided {sf[1]}/{sf[2]} rays differ {sf[4]}/{sf[3]}; "
              f"fused K5-K6 ratio {st[0]:.3g} undecided {st[1]} of {st[2]}, shadow rays differ {st[3]}/{st[2]}")
        assert all(v <= max(limit, FUSED_K6_UNDECIDED_MAX) * max(st[2], 1) for v in st[1].values()), st
        assert st[3] <= (0 if not self.fast else K8_DISAGREE_MAX * st[2]), st
        assert s7[1] <= K7_UNDECIDED_MAX * max(s7[2], 1) and sf[1] <= K7_UNDECIDED_MAX * max(sf[2], 1), (s7, sf)
        assert sf[4] <= (0 if not self.fast else K8_DISAGREE_MAX * sf[3]), sf
        assert s9[1] <= limit * max(s9[2], 1) and s10[1] <= limit * max(s10[2], 1)
        assert all(v <= limit * max(s6[2], 1) for v in s6[1].values()), s6[1]
        assert s8[1] <= K8_DISAGREE_MAX * s8[0], s8
        assert all(v <= limit * max(s5[2], 1) for v in s5[1].values()), s5[1]
        assert s5[4] <= K8_DISAGREE_MAX * s5[3], s5


def _run(gpu, blue_noise, scene, strict, fused, frames=13, moves=(3, 5, 8, 11), extra_lights=0, remove=9001, nmap=False, rows=None,
         inject_k7=None):
    ch = Chain(gpu, blue_noise, scene, strict, fused, nmap, rows)
    many_lights(ch.e, extra_lights)
    for f in range(1, frames + 1):
        if f in moves:
            ch.move(f)
        if f == 4:
            ch.e.insert_light(9001, scenes.LIGHT_POINT, scenes.point_light((0.2, 1.0, 0.3), 0.08, (3.0, 2.0, 1.0), 6.0))
        if f == 7:
            ch.e.insert_light(9001, scenes.LIGHT_POINT, scenes.point_light((-0.3, 0.8, 0.1), 0.08, (3.0, 2.0, 1.0), 6.0))
        if f == 10:
            ch.e.remove_light(remove)
        ch.frame(inject_k7=inject_k7 and inject_k7(f))
    return ch


@pytest.mark.parametrize("size", [(224, 126), (67, 45), (37, 29), (63, 45)])
@pytest.mark.parametrize("scene_name", ["cornell", "demo_level", "textured_room", "cornell_spots", "cornell_many_lights", "cornell_remap",
                                        "normal_mapped_room"])
@pytest.mark.parametrize("strict", [True, False], ids=["strict", "fast"])
def test_di_merge_and_resolve_within_float64_bound(gpu, blue_noise, strict, scene_name, size):
    """K5, K6, K7, K8, K9 and K10 in the unfused schedule, every pixel / texel / pair, frames 1-13 (both GI cycles) with the camera
    moving and a light inserted, moved and removed; 67x45 leaves columns outside the half grid; the half grid of 63x45 is 64 wide, so
    on alternate rows the last pair's lhs is off the screen (nothing written, no copy through) and its texel b lies at x = 63 (dropped);
    37x29 is smaller than the 128 px tap radius (K7's mirrored taps land outside the frame).  Many lights: 23, so K5 draws 16 of them; remap: the light removed is from the
    middle of the list, so K6 meets a remapped slot; the normal-mapped room shades with ST_OPT_NORMAL_MAPS, so the mapped normals feed
    K7's normal test and every pdf."""
    many = scene_name in ("cornell_many_lights", "cornell_remap")
    ch = _run(gpu, blue_noise, SCENES[scene_name](*size), strict, fused=False, extra_lights=MANY_LIGHTS if many else 0,
              remove=REMAP_REMOVED if scene_name == "cornell_remap" else 9001, nmap=scene_name == "normal_mapped_room")
    assert 1e-3 < ch.stats["K7"][0] <= 1 and Q.pick_tight_ok(ch.k7_tight), (ch.stats["K7"], ch.k7_tight)
    assert ch.stats["K9"][2] > 0 and 0 < ch.stats["K10"][0] <= 1 and 0 < ch.stats["K6"][0] <= 1 and ch.stats["K8"][0] > 0
    assert ch.k6_branches[0] > 0 and Q.tight_ok(ch.k6_tight), (ch.k6_branches, ch.k6_tight)
    if scene_name == "cornell_remap":
        assert ch.k6_branches[2] > 0, "no reprojected reservoir named the remapped slot"
    ch.report(f"{scene_name} {size} {'strict' if strict else 'fast'}")
    # the bound is not vacuous: most values are bounded tightly, and some error uses a visible part of its bound
    b, some = ch.bounds[-1]
    frac, n = Q.tight_fraction(list(b), some)
    assert n > 0 and frac >= 0.99, frac
    assert ch.k9_tight[1] > 0 and ch.k9_tight[0] >= 0.99 * ch.k9_tight[1], ch.k9_tight
    assert ch.stats["K10"][0] > 1e-3 and ch.stats["K9"][0] > 1e-3 and ch.stats["K6"][0] > 1e-3
    assert 1e-3 < ch.stats["K5"][0] <= 1 and ch.stats["K5"][3] > 0 and Q.sampling_tight_ok(ch.k5_tight), ch.k5_tight




def _empty_reservoirs(seed):
    """Sets M = 0 on half of di_reservoirs[1]'s pixels before K7 (or the fused K7 + K8 + K9): long walks, walks that reach the radius
    floor, accepted neighbours with an empty reservoir, and pairs whose lhs is empty while the rhs is not."""
    def inject(fr):
        rng = np.random.RandomState(seed)
        r = fr.e.read_buffer(fr.cam, "di_reservoirs_1").reshape(-1, 8).copy()
        r[rng.rand(len(r)) < 0.5, 0] = 0
        write_buffer(fr.e, fr.cam, "di_reservoirs_1", r.astype(np.float32))
    return inject


FUSED_CASES = [(s, size, False) for s in ("cornell", "demo_level", "textured_room", "cornell_spots")
               for size in ((224, 126), (67, 45), (63, 45))] + [("cornell", (67, 45), True)]


@pytest.mark.parametrize("scene_name,size,strict", FUSED_CASES,
                         ids=[f"{s}-{w}x{h}-{'strict' if t else 'fast'}" for s, (w, h), t in FUSED_CASES])
def test_di_resolve_product_default_within_bound(gpu, blue_noise, scene_name, size, strict):
    """The product default (fast build, fused passes): k_di_sample_temporal against K5 composed into K6 (every pixel; every third
    frame at 224x126), k_di_spatial_fused against K7, K8 and K9 composed (every pair), inputs read just before each launch, K10
    against its bound, and neither fused DI launch touches the scratch textures.  The small screens get empty reservoirs injected
    before the fused K7-K9 launch on every other frame; 63x45 has pairs whose lhs is off the screen and texel b at x = 63, which the
    launch does not trace.  The strict-build case calibrates the compositions: there every rebuilt shadow ray must agree."""
    w, h = size
    inject = (lambda f: _empty_reservoirs(f) if f % 2 == 0 else None) if w < 224 else None
    ch = _run(gpu, blue_noise, SCENES[scene_name](w, h), strict=strict, fused=True, inject_k7=inject)
    assert ch.stats["K9"][2] == 0 and ch.stats["K10"][2] > 0
    sf, st = ch.stats["K7-K9"], ch.stats["K5-K6"]
    assert sf[2] > 0 and sf[3] > 0 and 1e-3 < sf[0] <= 1, sf
    assert st[2] > 0 and 1e-3 < st[0] <= 1, st
    ch.report(f"{scene_name} {w}x{h} product default{' (strict)' if strict else ''}")


def test_di_resolve_1080p_product_default(gpu, blue_noise):
    """Two product-default frames at 1080p: K10 on every pixel, the fused K7 + K8 + K9 launch on a band of 32 rows (the fused K5 + K6
    launch is checked at the smaller sizes above; here only that it leaves the scratch textures alone)."""
    ch = _run(gpu, blue_noise, scenes.cornell(1920, 1080), strict=False, fused=True, frames=2, moves=(), rows=np.arange(524, 556))
    assert ch.stats["K7-K9"][2] > 0
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


def _temporal_edges(seed):
    """Rewrites K6's inputs: in di_reservoirs[0] M at 63, 64, 65 and 1e6 and w at 0, a denormal and 1e6; in the reprojection map,
    previous positions at exact .5 fractions (round half away from zero) and on the last row and column.  No position is moved
    outside the frame: frame reprojection never produces one, and the reference would read outside its buffers."""
    def inject(fr):
        rng = np.random.RandomState(seed)
        r = fr.e.read_buffer(fr.cam, "di_reservoirs_0").reshape(-1, 8).copy()
        live = r[:, 0] > 0
        k = rng.randint(0, 8, len(r))
        r[:, 0] = np.where(live & (k == 1), 63, np.where(live & (k == 2), 64, np.where(live & (k == 3), 65, np.where(live & (k == 4), 1e6, r[:, 0]))))
        r[:, 1] = np.where(live & (k == 5), 0, np.where(live & (k == 6), np.float32(1e-41), np.where(live & (k == 7), 1e6, r[:, 1])))
        write_buffer(fr.e, fr.cam, "di_reservoirs_0", r.astype(np.float32))
        m = fr.read("reprojection_map").copy()
        some = m[..., 2] > 0
        j = rng.randint(0, 5, some.shape)
        half = lambda v, n: np.minimum(np.floor(v), n - 2) + np.float32(0.5)     # rounds up to at most n - 1
        m[..., 0] = np.where(some & (j == 1), half(m[..., 0], fr.w), np.where(some & (j == 3), fr.w - 1, m[..., 0]))
        m[..., 1] = np.where(some & (j == 2), half(m[..., 1], fr.h), np.where(some & (j == 4), fr.h - 1, m[..., 1]))
        fr.write("reprojection_map", m)
    return inject


MANY_LIGHTS = 21        # with Cornell's point light and the sun: 23 lights, so K5 draws 16 of them and `% light_count` is not trivial
REMAP_REMOVED = 9210    # a light from the middle of that list: removing it remaps the last slot as well as killing its own


def many_lights(engine, n):
    """n small point lights on a ring under the Cornell box's ceiling, handles 9200 + i."""
    for i in range(n):
        a = 2 * np.pi * i / max(n, 1)
        engine.insert_light(9200 + i, scenes.LIGHT_POINT, scenes.point_light((0.7 * np.cos(a), 1.6 + 0.1 * (i % 3), 0.7 * np.sin(a)),
                                                                             0.03, (0.4 + 0.1 * (i % 4), 0.5, 0.6 - 0.1 * (i % 3)), 4.0))


@pytest.mark.parametrize("strict", [True, False], ids=["strict", "fast"])
@pytest.mark.parametrize("scene_name", ["cornell", "cornell_spots"])
def test_di_edge_inputs_within_bound(gpu, blue_noise, strict, scene_name):
    """Edge contents injected before K6 (last frame's M around the clamp of 64 and far past it, w 0 / denormal / 1e6, reprojected
    positions on .5 fractions and on the last row and column), before K9 (M at the cap region and far past it, w 0 / denormal / 1e6,
    pdf 0) and before K10 (metallic and reflectance bytes 0 / 255, roughness byte 0, normals along the view direction at minimum
    roughness), with the edge lights and the camera moving.  The light table is filled up to K5's boundaries: 16 lights on Cornell,
    where max_samples = min(light_count, 16) first reaches its cap, and 17 with the spot lights, the first count past it, where
    `% light_count` leaves some lights undrawn (23, further past it, is the many-lights scene run)."""
    scene = SCENES[scene_name](67, 45)
    ch = Chain(gpu, blue_noise, scene, strict, fused=False)
    edge_lights(ch.e)
    want = EDGE_LIGHT_COUNT[scene_name]
    many_lights(ch.e, want - (len(scene["lights"]) + 1 + 4))       # + the sun and the four edge lights
    for f in range(1, 6):
        if f in (2, 4):
            ch.move(f)
        ch.frame(_reservoir_edges(10 * f), _gbuffer_edges(10 * f + 1, ch), _temporal_edges(10 * f + 2), _empty_reservoirs(10 * f + 3))
        assert ch.e.read_scene("world")[:1].view(np.uint32)[0] == want
    assert 0 < ch.stats["K5"][0] <= 1 and ch.stats["K5"][2] > 0
    # with half the reservoirs empty every branch of K7's walk is taken
    assert all(v > 0 for v in ch.k7_branches.values()), ch.k7_branches
    ch.report(f"edges {scene_name} {want} lights {'strict' if strict else 'fast'}", UNDECIDED_MAX_EDGES)


EDGE_LIGHT_COUNT = {"cornell": 16, "cornell_spots": 17}


def test_fast_shading_build_is_not_strict(gpu, blue_noise):
    """The fast-tier runs above really ran the fast build: the same inputs through the strict K5, K6, K9 and K10 give different bits
    somewhere in each pass's output."""
    from strolle_b200.engine import OPT_SHADING_FAST_MATH
    e = _engine(gpu, blue_noise, False, False)
    cam = scenes.apply(e, scenes.cornell(67, 45))
    for _ in range(2):
        e.tick(); e.render_camera(cam)
    e.tick()
    fr = Frame(e, cam, 67, 45)
    k5, k6, k9, k10 = fr.steps(P_DI_SAMPLING)[0], fr.steps(P_DI_TEMPORAL)[0], fr.steps(P_DI_SPATIAL_SAMPLE)[0], fr.steps(P_DI_RESOLVING)[0]
    fr.run_to(k5 - 1)
    pre5 = e.read_buffer(cam, "di_reservoirs_1").copy()      # K5 reads the G-buffer, the lights and the blue noise; it writes this
    fr.run_to(k5)
    fast5 = e.read_buffer(cam, "di_reservoirs_1").copy()
    fr.run_to(k6 - 1)
    pre6 = {n: e.read_buffer(cam, n).copy() for n in ("di_reservoirs_0", "di_reservoirs_1")}   # K6's reservoir inputs
    fr.run_to(k6)
    fast6 = e.read_buffer(cam, "di_reservoirs_1").copy()
    fr.run_to(k9)                        # K9 reads di_reservoirs[1] and the stash, which it leaves as they were
    fast9 = e.read_buffer(cam, "di_reservoirs_2").copy()
    fr.run_to(k10)                       # K10 reads di_reservoirs[2] and the G-buffer; it writes di_reservoirs[0]
    fast10 = fr.read("di_spec_samples").copy(), fr.read("di_diff_samples").copy()
    e.set_option(OPT_SHADING_FAST_MATH, 0)
    e.render_range(cam, k10, k10)
    strict10 = fr.read("di_spec_samples"), fr.read("di_diff_samples")
    e.render_range(cam, k9, k9)
    strict9 = e.read_buffer(cam, "di_reservoirs_2")
    assert (fast9.view(np.uint32) != strict9.view(np.uint32)).any(), "K9"
    assert any((a.view(np.uint32) != b.view(np.uint32)).any() for a, b in zip(fast10, strict10)), "K10"

    def rerun_k6(fast):
        """K6 again on its own inputs: last frame's reservoirs (which K10 has since overwritten) and K5's samples (which K6 updates
        in place) are put back first."""
        for n, a in pre6.items():
            write_buffer(e, cam, n, a)
        e.set_option(OPT_SHADING_FAST_MATH, int(fast))
        e.render_range(cam, k6, k6)
        return e.read_buffer(cam, "di_reservoirs_1").copy()
    strict6 = rerun_k6(False)
    # the inputs are restored completely: the fast K6 run again gives its first result bit for bit
    assert (rerun_k6(True).view(np.uint32) == fast6.view(np.uint32)).all(), "K6 re-run on restored inputs"
    assert (fast6.view(np.uint32) != strict6.view(np.uint32)).any(), "K6"

    def rerun_k5(fast):
        write_buffer(e, cam, "di_reservoirs_1", pre5)
        e.set_option(OPT_SHADING_FAST_MATH, int(fast))
        e.render_range(cam, k5, k5)
        return e.read_buffer(cam, "di_reservoirs_1").copy()
    strict5 = rerun_k5(False)
    assert (rerun_k5(True).view(np.uint32) == fast5.view(np.uint32)).all(), "K5 re-run on restored inputs"
    assert (fast5.view(np.uint32) != strict5.view(np.uint32)).any(), "K5"


# ---- the fast build's elementary functions ------------------------------------------------------------------------------------

def test_fast_elementary_functions_within_assumed_constants(gpu, blue_noise):
    """sin / cos (__sincosf), exp (__expf), pow (__powf), sqrt (sqrt.approx), division (div.full), acos and atan2 of the fast-shading
    build, measured on the argument ranges the ReSTIR kernels and the sky use, within the constants a bound on them assumes
    (tests/ref64_restir.py)."""
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
    # acos on all of [-1, 1] (densely toward +-1: the sky's zenith angle and horizon), atan2 of points of every angle at radii 1e-3 to
    # 1.26 (the sky's azimuth)
    xa = np.concatenate([np.linspace(-1.0, 1.0, 400001), 1 - np.logspace(-8, 0, 10 ** 5), np.logspace(-8, 0, 10 ** 5) - 1]).astype(np.float32)
    xa = xa[np.abs(xa) <= 1]
    err_a = np.abs(e.device_math("acos_fast", xa) - np.arccos(xa.astype(np.float64))).max()
    ang, rad = rng.uniform(0, 2 * np.pi, 10 ** 6), 10 ** rng.uniform(-3, 0.1, 10 ** 6)
    ys, xs2 = (rad * np.sin(ang)).astype(np.float32), (rad * np.cos(ang)).astype(np.float32)
    err_t = np.abs(e.device_math("atan2_fast", ys, xs2) - np.arctan2(ys.astype(np.float64), xs2.astype(np.float64))).max()
    print(f"\nfast elementary functions: sin {err_s:.3g} cos {err_c:.3g} acos {err_a:.3g} atan2 {err_t:.3g} (abs), exp {rel_e:.3g}, "
          f"pow {rel_p:.3g}, sqrt {rel_q:.3g}, div {rel_d:.3g} (rel)")
    assert err_a <= Q.ACOS_ABS_FAST and err_t <= Q.ATAN2_ABS_FAST
    assert err_s <= Q.SIN_ABS_FAST and err_c <= Q.SIN_ABS_FAST
    assert rel_e <= Q.EXP_REL_FAST and rel_p <= Q.POW_REL_FAST
    assert rel_q <= Q.SQRT_REL_FAST and rel_d <= Q.DIV_REL
    # and they are the approximations, not the strict kernels
    assert (e.device_math("sin_fast", x) != e.device_math("sin", x)).any()
