"""Environment-map sampling (ST_OPT_ENVIRONMENT_MAP_SAMPLING): the distribution against its numpy restatement, the density against
float64 quadrature, the draws against the density (chi-squared, cell by cell), K12's mixture, support, known answers, the extension's
deliberate mistakes and the variance it removes; on the GPU, the device against the extension (the distribution, every camera buffer of
the strict tier, the product tier), the option's no-op cases, the distribution's life cycle, row strips, and the frame mean."""
import math

import numpy as np
import pytest
from scipy import stats

from strolle_b200 import scenes
from oracle_envmap import pyoracle_envmap as E
from tests import ref64_envsample as R
from tests.util import CAMERA_BUFFERS, assert_bits_equal, rel_l2

OPT_ENVIRONMENT_MAP_SAMPLING = 19
STAT_ENVIRONMENT_MAP_LAUNCHES, STAT_ENVIRONMENT_MAP_DISTRIBUTION_BUILDS = 13, 14
OPT_NORMAL_MAPS, OPT_LIGHT_GRID, OPT_TEXTURE_FILTER = 14, 16, 17


def _block_map(w=64, h=32):
    """Black except for one bright block (rows 8..10, columns 20..23), high in the sky."""
    m = np.zeros((h, w, 4), np.float32)
    m[8:11, 20:24, :3] = (40.0, 30.0, 20.0)
    return m


def _single_texel_map(w=48, h=24, at=(7, 0)):
    m = np.zeros((h, w, 4), np.float32)
    m[at[0], at[1], :3] = (1000.0, 500.0, 100.0)
    return m


MAPS = {
    "courtyard_sky": lambda: scenes.courtyard_sky(),
    "sunlit_sky": lambda: scenes.sunlit_sky(),
    "1x1": lambda: np.full((1, 1, 4), 2.5, np.float32),
    "1xN": lambda: np.random.RandomState(4).uniform(0, 3, (1, 37, 4)).astype(np.float32),
    "Nx1": lambda: np.random.RandomState(5).uniform(0, 3, (29, 1, 4)).astype(np.float32),
    "odd": lambda: np.random.RandomState(6).exponential(1.0, (13, 37, 4)).astype(np.float32),
    "single_texel": lambda: _single_texel_map(),
}


def _xi(n, seed):
    """n draws of (xi1, xi2) as rng_f makes them: a u32 times 2^-32, rounded to f32."""
    r = np.random.RandomState(seed).randint(0, 2 ** 32, size=(n, 2), dtype=np.uint64)
    return (r.astype(np.float32) * np.float32(2.0 ** -32)).astype(np.float32)


# ---- CPU ------------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", sorted(MAPS))
def test_distribution_matches_numpy(name):
    """The extension's CDFs (the device's rule) are np.cumsum's over the float32 weights, bit for bit."""
    tex = MAPS[name]()
    W, H, total, marg, cond = E.EnvMap(tex).distribution()
    m, c, t = R.cdfs(tex)
    assert (W, H) == (tex.shape[1], tex.shape[0])
    assert_bits_equal(marg, m, "marginal"); assert_bits_equal(cond, c, "conditional"); assert_bits_equal(total, t, "total")


@pytest.mark.parametrize("name", ["courtyard_sky", "odd", "single_texel", "1xN", "Nx1"])
def test_pdf_integrates_to_one(name):
    """The float64 restatement of env_pdf integrates to 1 +- 1e-3 over the sphere (midpoint quadrature, 8 x 8 points per cell and at
    least 1024 x 512 in all), at rotation 0 and 2.5; so does the extension's f32 env_pdf."""
    tex = MAPS[name]()
    marg, cond, _ = R.cdfs(tex)
    prob = R.cell_probabilities(marg, cond)
    H, W = prob.shape
    d, dw, _, _ = R.sphere_grid(max(8 * W, 1024), max(8 * H, 512))
    for rot in (0.0, 2.5):
        assert abs((R.env_pdf64(prob, rot, d) * dw).sum() - 1.0) < 1e-3
        em = E.EnvMap(tex, rotation=rot)
        assert abs((em.pdf(d).astype(np.float64) * dw).sum() - 1.0) < 1e-3


@pytest.mark.parametrize("name", ["courtyard_sky", "odd", "single_texel", "1xN"])
def test_draws_have_the_density_of_their_cell(name):
    """For every env_draw output, env_pdf is the density of the cell it was drawn from, except where the f32 direction rounds onto a
    neighbouring cell: there it is that cell's density.  Such draws are under 0.1%.  The tolerance is relative 1e-5 + 1e-7 / sin^2
    theta: env_pdf's f32 sin theta = sqrt(1 - y^2) loses up to 3e-8 / sin^2 theta to the rounding of y^2 near the poles."""
    tex = MAPS[name]()
    em = E.EnvMap(tex, rotation=1.0)
    d, cells = em.draw(_xi(200000, 1))
    p = em.pdf(d).astype(np.float64)
    _, _, _, marg, cond = em.distribution()
    prob = R.cell_probabilities(marg, cond)
    H, W = prob.shape
    st = np.sqrt(np.maximum(0.0, 1.0 - d[:, 1].astype(np.float64) ** 2))
    want = prob[cells[:, 0], cells[:, 1]] * W * H / (2 * math.pi ** 2 * st)
    tol = 1e-5 + 1e-7 / st ** 2
    ok = (np.abs(p - want) <= tol * want) | ((p == want) & np.isinf(p))
    assert (~ok).mean() < 1e-3, (~ok).mean()
    near = np.zeros((~ok).sum(), bool)
    for di in (-1, 0, 1):
        for dj in (-1, 0, 1):
            i = np.clip(cells[~ok, 0].astype(int) + di, 0, H - 1); j = (cells[~ok, 1].astype(int) + dj) % W
            want = prob[i, j] * W * H / (2 * math.pi ** 2 * st[~ok])
            near |= np.abs(p[~ok] - want) <= tol[~ok] * want
    assert near.all()


def _chi2(counts, expected):
    """Chi-squared p-value over bins with at least 5 expected draws (the rest pooled into one bin)."""
    big = expected >= 5
    c = np.concatenate([counts[big], [counts[~big].sum()]]); e = np.concatenate([expected[big], [expected[~big].sum()]])
    keep = e > 0
    return stats.chisquare(c[keep], e[keep] * c[keep].sum() / e[keep].sum()).pvalue


@pytest.mark.parametrize("name", ["courtyard_sky", "odd", "sunlit_sky"])
def test_draws_chi_squared(name):
    """10^6 draws, binned by the cell of the drawn direction (float64 u, v at rotation 0.7), follow the cell probabilities
    (chi-squared p > 1e-3)."""
    tex = MAPS[name]()
    em = E.EnvMap(tex, rotation=0.7)
    d, _ = em.draw(_xi(1000000, 2))
    marg, cond, _ = R.cdfs(tex)
    prob = R.cell_probabilities(marg, cond)
    H, W = prob.shape
    u, v = R.uv64(d, float(np.float32(0.7)))
    i = np.clip(np.floor(v * H).astype(int), 0, H - 1); j = np.floor(u * W).astype(int) % W
    counts = np.bincount(i * W + j, minlength=H * W).astype(np.float64)
    assert _chi2(counts, prob.ravel() * len(d)) > 1e-3


SURF_N, SURF_V = np.array([0.0, 1.0, 0.0]), np.array([0.3, 0.8, 0.5]) / np.linalg.norm([0.3, 0.8, 0.5])


@pytest.mark.parametrize("metallic,roughness", [(0.0, 0.5), (0.5, 0.3), (1.0, 0.1)])
def test_mixture_chi_squared(metallic, roughness):
    """K12's one-sample mixture: 10^6 directions (one WhiteNoise each, as K12 draws them) binned on a 32 x 16 (u, v) grid follow
    q = 1/2 p_bsdf + 1/2 p_env integrated by float64 quadrature over 4096 x 2048 points (chi-squared p > 1e-3), and the q / kappa
    the extension returns is the float64 one (relative 1e-4) for 99.9% of the draws where kappa > 0.  The reference's GGX sampler sends every half vector
    with h.v <= 0 to -v (its reflection clamps h.v to 0); those draws, where kappa = 0 and the candidate carries w = 0, are left out,
    as is their mass from q's integral (1 - q's integral is that share)."""
    tex = scenes.courtyard_sky()
    em = E.EnvMap(tex)
    seeds = np.random.RandomState(7).randint(0, 2 ** 32, 1000000, dtype=np.uint64).astype(np.uint32)
    rec = em.surface_draws(False, SURF_N, SURF_V, metallic, roughness, seeds)
    atom = np.linalg.norm(rec[:, :3] + SURF_V[None, :].astype(np.float32), axis=1) < 1e-5
    assert not np.isfinite(rec[atom, 3]).any()
    rec = rec[~atom]
    d = rec[:, :3].astype(np.float64)
    marg, cond, _ = R.cdfs(tex)
    prob = R.cell_probabilities(marg, cond)
    gd, gw, gu, gv = R.sphere_grid(4096, 2048)
    q, _ = R.mixture64(prob, 0.0, SURF_N, SURF_V, metallic, np.float32(roughness), gd)
    assert abs((q * gw).sum() - (1.0 - atom.mean())) < 2e-3
    bins = np.floor(gv * 16).astype(int) * 32 + np.floor(gu * 32).astype(int)
    expected = np.bincount(bins, weights=q * gw, minlength=512) * len(d)
    u, v = R.uv64(d, 0.0)
    got = np.bincount(np.clip(np.floor(v * 16).astype(int), 0, 15) * 32 + np.floor(u * 32).astype(int) % 32, minlength=512)
    assert _chi2(got.astype(np.float64), expected) > 1e-3
    qd, kd = R.mixture64(prob, 0.0, SURF_N, SURF_V, metallic, np.float32(roughness), d)
    pos = (kd > 0) & np.isfinite(rec[:, 3])
    assert pos.mean() > 0.5
    close = np.isclose(rec[pos, 3], qd[pos] / kd[pos], rtol=1e-4, atol=0.0)
    assert close.mean() > 0.999, close.mean()   # the rest: f32 u, v on the far side of a cell edge, or f32 sin theta at a pole


def test_support_covers_the_lookup():
    """Every direction whose lookup is non-zero has env_pdf > 0: around an isolated bright texel (away from and on the u = 0 / 1 seam)
    and across the seam, at rotations 0 and 1.3, on a grid of 400 x 400 directions spanning the texel's neighbourhood."""
    for at in ((7, 20), (7, 0), (12, 47)):
        tex = _single_texel_map(at=at)
        H, W = tex.shape[:2]
        for rot in (0.0, 1.3):
            em = E.EnvMap(tex, rotation=rot)
            v = (at[0] + np.linspace(-2.5, 3.5, 400)) / H
            u = (at[1] + np.linspace(-2.5, 3.5, 400)) / W
            uu, vv = np.meshgrid(u, v)
            theta, phi = vv.ravel() * math.pi, (uu.ravel() - 0.5) * 2 * math.pi - rot
            d = np.stack([np.sin(theta) * np.sin(phi), np.cos(theta), -np.sin(theta) * np.cos(phi)], 1).astype(np.float32)
            lit = em.sample(d).max(axis=1) > 0
            assert lit.sum() > 100
            assert (em.pdf(d)[lit] > 0).all()


N_KNOWN = 1000000   # draws per known answer


def _k12_k13_means(em, seeds, metallic=0.0, roughness=0.5):
    """The K12 initial sample on an open plane (every upward bounce misses: radiance = the map, weight kappa / q), and K13's
    sky-draw value over its probability of 0.25, averaged over the draws (luminance-free: channel 0)."""
    a = em.surface_draws(False, SURF_N, SURF_V, metallic, roughness, seeds)
    w = np.where(np.isfinite(a[:, 3]) & (a[:, 3] > 0), 1.0 / a[:, 3].astype(np.float64), 0.0)
    b = em.surface_draws(True, SURF_N, SURF_V, metallic, roughness, seeds)
    return (a[:, 4] * w).mean(), (b[:, 4].astype(np.float64) / 0.25).mean()


def _block_quadrature(tex, rot, metallic=0.0, roughness=0.5):
    """float64 quadrature (4096 x 2048) of int L kappa and of int L cos+ / (2 pi) / 0.25 for the block map."""
    d, dw, _, _ = R.sphere_grid(4096, 2048)
    L = E.EnvMap(tex, rotation=rot).sample(d.astype(np.float32))[:, 0].astype(np.float64)
    marg, cond, _ = R.cdfs(tex)
    _, kappa = R.mixture64(R.cell_probabilities(marg, cond), rot, SURF_N, SURF_V, metallic, np.float32(roughness), d)
    cos = np.maximum(d @ SURF_N, 0.0)
    return (L * kappa * dw).sum(), (L * cos * dw).sum() / (2 * math.pi) / 0.25


def test_known_answers():
    """A constant map c, m = 0: the mean of K12's missed-bounce radiance x w is pi c and K13's sky-draw value (over 0.25) has mean
    2 c, each within 0.5%.  A map black except for one bright block (m = 0 and m = 0.5): the mean of K12's initial sample is the
    float64 quadrature of int L kappa within 1%, and K13's the quadrature of int L cos / 2 pi / 0.25 within 1%; 10^6 draws each."""
    seeds = np.random.RandomState(8).randint(0, 2 ** 32, N_KNOWN, dtype=np.uint64).astype(np.uint32)
    c = 1.7
    k12, k13 = _k12_k13_means(E.EnvMap(np.full((16, 32, 4), c, np.float32)), seeds)
    assert abs(k12 / (math.pi * c) - 1) < 5e-3 and abs(k13 / (2 * c) - 1) < 5e-3, (k12, k13)
    tex = _block_map()
    rot = float(np.float32(1.0))
    for metallic, roughness in ((0.0, 0.5), (0.5, 0.3)):
        k12, k13 = _k12_k13_means(E.EnvMap(tex, rotation=1.0), seeds, metallic, roughness)
        q12, q13 = _block_quadrature(tex, rot, metallic, roughness)
        assert abs(k12 / q12 - 1) < 0.01 and abs(k13 / q13 - 1) < 0.01, (metallic, k12, q12, k13, q13)


def _mutation_checks(mutation):
    """The bounds a deliberate mistake can leave: the CDFs against numpy, the f32 density's integral, and the block map's known
    answers (m = 0.5, rotation 1)."""
    tex = _block_map()
    em = E.EnvMap(tex, rotation=1.0, mutation=mutation)
    _, _, total, marg, cond = em.distribution()
    m, c, _ = R.cdfs(tex)
    cdf_ok = (marg.view(np.uint32) == m.view(np.uint32)).all() and (cond.view(np.uint32) == c.view(np.uint32)).all()
    d, dw, _, _ = R.sphere_grid(1024, 512)
    pdf_ok = abs((em.pdf(d.astype(np.float32)).astype(np.float64) * dw).sum() - 1.0) < 1e-3
    seeds = np.random.RandomState(9).randint(0, 2 ** 32, N_KNOWN, dtype=np.uint64).astype(np.uint32)
    k12, k13 = _k12_k13_means(em, seeds, 0.5, 0.3)
    q12, q13 = _block_quadrature(tex, float(np.float32(1.0)), 0.5, 0.3)
    return dict(cdf=cdf_ok, pdf=pdf_ok, k12=abs(k12 / q12 - 1) < 0.01, k13=abs(k13 / q13 - 1) < 0.01)


def test_without_mistakes_every_bound_holds():
    assert all(_mutation_checks(None).values())


@pytest.mark.parametrize("mutation", sorted(E.SAMPLING_MUTATIONS))
def test_mutation_leaves_a_bound(mutation):
    """Each deliberate mistake (no 3 x 3 max, no sin theta in the weights or in the density, the draw's rotation reversed or its v
    flipped, the drawn component's pdf in place of the mixture's, kappa dropped) leaves at least one bound."""
    checks = _mutation_checks(mutation)
    assert not all(checks.values()), checks


def test_variance_lower_on_sunlit_sky():
    """The variance of the K12 initial sample (missed bounce: L w) and of K13's sky-draw value (over 0.25) at an open, upward-facing
    diffuse surface under sunlit_sky (1024 x 512), by float64 quadrature over 4096 x 2048 directions of each estimator's second
    moment under the density it draws from: at least 4x lower with the option on.  (A frame-based estimate at test sizes cannot see
    the option-off fireflies: a 0.5 degree sun is hit by about one uniform draw in 10^5.)"""
    tex = scenes.sunlit_sky(1024, 512)
    d, dw, _, _ = R.sphere_grid(4096, 2048)
    L = E.EnvMap(tex).sample(d.astype(np.float32)).astype(np.float64) @ np.array([0.2126, 0.7152, 0.0722])
    marg, cond, _ = R.cdfs(tex)
    pe = R.env_pdf64(R.cell_probabilities(marg, cond), 0.0, d)
    n = np.array([0.0, 1.0, 0.0])
    cos = d @ n
    up = cos > 0
    hemi = up / (2 * math.pi)   # the uniform hemisphere's density
    def var(value, density):
        keep = density > 0
        m1 = (value * density * dw)[keep].sum()
        return (value[keep] ** 2 * density[keep] * dw[keep]).sum() - m1 * m1, m1
    v12_off, m12_off = var(math.pi * L, hemi)
    q, kappa = R.mixture64(R.cell_probabilities(marg, cond), 0.0, n, SURF_V, 0.0, np.float32(0.5), d)
    with np.errstate(divide="ignore", invalid="ignore"):
        v12_on, m12_on = var(np.where(q > 0, L * kappa / q, 0.0), q)
        v13_off, m13_off = var(L * cos / 0.25, hemi)
        v13_on, m13_on = var(np.where(up & (pe > 0), L * np.maximum(cos, 0) / (2 * math.pi * pe) / 0.25, 0.0), pe)
    print(f"sunlit_sky variance: K12 off {v12_off:.4g} on {v12_on:.4g} (factor {v12_off / v12_on:.3g}); "
          f"K13 off {v13_off:.4g} on {v13_on:.4g} (factor {v13_off / v13_on:.3g})")
    assert abs(m12_on / m12_off - 1) < 2e-3 and abs(m13_on / m13_off - 1) < 2e-3
    assert v12_off >= 4 * v12_on and v13_off >= 4 * v13_on


def test_option_validation_in_extension():
    eo = E.EnvMapOracleEngine()
    for bad in (-1, 2, 7):
        with pytest.raises(ValueError):
            eo.set_option(OPT_ENVIRONMENT_MAP_SAMPLING, bad)


# ---- GPU ------------------------------------------------------------------------------------------------------------------------

def _gpu(blue_noise, exact=True, fused=None, sampling=True, options=None):
    import strolle_b200
    from strolle_b200.engine import OPT_FUSED_PASSES
    e = strolle_b200.Engine(blue_noise=blue_noise, exact=exact)
    if fused is not None:
        e.set_option(OPT_FUSED_PASSES, int(fused))
    if sampling:
        e.set_option(OPT_ENVIRONMENT_MAP_SAMPLING, 1)
    for k, v in (options or {}).items():
        e.set_option(k, v)
    return e


def _moving_step(engines, scene, f, w, h):
    """Frame f: env_courtyard orbits its camera and slides the crate; env_sunlit pans its camera a little.  Then tick and render."""
    c = scene["camera"]
    if scene["name"] == "env_courtyard":
        xf, crate = scenes.env_courtyard_motion(f)
    else:
        xf, crate = np.asarray(c["transform"], np.float32).reshape(4, 4).copy(), None
        xf[3, :3] += np.array([0.03 * f, 0.0, -0.02 * f], np.float32)
        xf = xf.reshape(-1)
    for e, cam in engines:
        e.update_camera(cam, c["mode"], c["denoise"], c["ref_depth"], w, h, xf, c["projection"])
        if crate is not None:
            e.insert_instance(334, 234, 133, crate)
        e.tick(); e.render_camera(cam)


def _scene(name, w, h):
    sc = scenes.env_sunlit(w, h) if name == "env_sunlit" else scenes.env_courtyard(w, h)
    sc["environment_map"] = dict(sc["environment_map"], rotation=2.5)
    return sc


@pytest.mark.gpu
def test_device_distribution_matches_numpy(blue_noise):
    """The device's CDFs, as st_read_scene("environment_map_distribution") returns them, are numpy's bit for bit (courtyard_sky,
    sunlit_sky, an odd size, 1 x 1, one bright texel); each new map is one build."""
    from strolle_b200.engine import StrolleError
    e = _gpu(blue_noise)
    scenes.apply(e, scenes.env_courtyard(32, 18))
    for k, name in enumerate(("courtyard_sky", "sunlit_sky", "odd", "1x1", "single_texel")):
        tex = MAPS[name]()
        e.set_environment_map(tex, 1.0, 0.0); e.tick()
        W, H, total, marg, cond = E.parse_distribution(e.read_scene("environment_map_distribution"))
        m, c, t = R.cdfs(tex)
        assert (W, H) == (tex.shape[1], tex.shape[0])
        assert_bits_equal(marg, m, name); assert_bits_equal(cond, c, name); assert_bits_equal(total, t, name)
        assert e.get_stat(STAT_ENVIRONMENT_MAP_DISTRIBUTION_BUILDS) == k + 1
    e.set_option(OPT_ENVIRONMENT_MAP_SAMPLING, 0); e.tick()
    with pytest.raises(StrolleError):
        e.read_scene("environment_map_distribution")
    for bad in (-1, 2):
        with pytest.raises(StrolleError):
            e.set_option(OPT_ENVIRONMENT_MAP_SAMPLING, bad)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["env_sunlit", "env_courtyard"])
@pytest.mark.parametrize("size", [(224, 126), (67, 45)])
def test_strict_tier_bit_exact_with_extension(blue_noise, name, size):
    """The option on, strict arithmetic, 13 moving frames, the unfused and fused schedules: every camera buffer is the extension's,
    bit for bit (the fused schedule: every buffer it still writes)."""
    from tests.test_gpu_parity import NOT_WRITTEN_WHEN_FUSED
    w, h = size
    scene = _scene(name, w, h)
    gs = [_gpu(blue_noise, True, fused=fused) for fused in (False, True)]
    cams = [scenes.apply(g, scene) for g in gs]
    eo = E.EnvMapOracleEngine(blue_noise=blue_noise)
    eo.set_option(OPT_ENVIRONMENT_MAP_SAMPLING, 1)
    co = scenes.apply(eo, scene)
    for f in range(13):
        _moving_step([(g, c) for g, c in zip(gs, cams)] + [(eo, co)], scene, f, w, h)
        assert eo.sampled
        for fused, g, c in zip((False, True), gs, cams):
            for n in CAMERA_BUFFERS:
                if fused and n in NOT_WRITTEN_WHEN_FUSED:
                    continue
                assert_bits_equal(g.read_buffer(c, n), eo.read_buffer(co, n), f"{name} fused={fused} {size} frame {f + 1} {n}")
    assert all(g.get_stat(STAT_ENVIRONMENT_MAP_DISTRIBUTION_BUILDS) == 1 for g in gs)


@pytest.mark.gpu
def test_with_other_options_fused_is_unfused(blue_noise):
    """The option on with normal maps, texture filtering and the light grid: the fused K12 + K13 launch gives the unfused frames bit
    for bit in every buffer it writes (the ENV_SAMPLED instantiations compose with NMAP, TEXF and LGRID), and K12 and K13 differ from
    the option-off run."""
    from tests.test_gpu_parity import NOT_WRITTEN_WHEN_FUSED
    w, h = 224, 126
    sc = _scene("env_courtyard", w, h)
    sc["lights"] = list(sc["lights"]) + [(431, scenes.LIGHT_POINT, scenes.point_light((1.0, 1.0, 2.0), 0.1, (1.0, 1.0, 1.0), 15.0))]
    opts = {OPT_NORMAL_MAPS: 1, OPT_TEXTURE_FILTER: 1, OPT_LIGHT_GRID: 8}
    es = [_gpu(blue_noise, True, fused=fz, options=opts) for fz in (False, True)] + [_gpu(blue_noise, True, fused=False, sampling=False, options=opts)]
    cs = [scenes.apply(e, sc) for e in es]
    for f in range(5):
        _moving_step(list(zip(es, cs)), sc, f, w, h)
        for n in CAMERA_BUFFERS:
            if n not in NOT_WRITTEN_WHEN_FUSED:
                assert_bits_equal(es[1].read_buffer(cs[1], n), es[0].read_buffer(cs[0], n), f"frame {f + 1} {n}")
    assert (es[0].read_buffer(cs[0], "gi_reservoirs_1") != es[2].read_buffer(cs[2], "gi_reservoirs_1")).any()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["env_sunlit", "env_courtyard"])
def test_product_tier_within_tolerance_of_extension(blue_noise, name):
    """The option on, product defaults: the G-buffer is the strict tier's bit for bit, and the composed frame stays within
    max(1e-3, 1.5 x the option-off drift) relative per-channel L2 of the extension over 13 frames."""
    w, h = 224, 126
    worst = {}
    for sampling in (True, False):
        scene = _scene(name, w, h)
        prod, strict = _gpu(blue_noise, False, sampling=sampling), _gpu(blue_noise, True, sampling=sampling)
        cp, cs = scenes.apply(prod, scene), scenes.apply(strict, scene)
        eo = E.EnvMapOracleEngine(blue_noise=blue_noise)
        eo.set_option(OPT_ENVIRONMENT_MAP_SAMPLING, int(sampling))
        co = scenes.apply(eo, scene)
        worst[sampling] = 0.0
        for f in range(13):
            _moving_step([(prod, cp), (strict, cs), (eo, co)], scene, f, w, h)
            for n in ("prim_gbuffer_d0_a", "prim_gbuffer_d0_b", "prim_gbuffer_d1_a", "prim_gbuffer_d1_b", "prim_triangle_ids"):
                assert_bits_equal(prod.read_buffer(cp, n), strict.read_buffer(cs, n), f"frame {f + 1} {n}")
            a = prod.read_buffer(cp, "output").reshape(-1, 4)[:, :3]
            b = eo.read_buffer(co, "output").reshape(-1, 4)[:, :3]
            for ch in range(3):
                worst[sampling] = max(worst[sampling], rel_l2(a[:, ch], b[:, ch]))
    print(f"{name}: worst relative L2 with sampling {worst[True]:.3g}, without {worst[False]:.3g}")
    assert worst[True] <= max(1e-3, 1.5 * worst[False])


@pytest.mark.gpu
def test_no_op_cases_are_bit_identical(blue_noise):
    """Option on with no map, and option on with an all-black map: every camera buffer is the option-off frame's, bit for bit, over 6
    moving frames; the black map's distribution is built (total 0) and not used."""
    w, h = 96, 54
    for kind in ("none", "black"):
        scene = _scene("env_courtyard", w, h)
        if kind == "none":
            del scene["environment_map"]
        else:
            scene["environment_map"] = dict(rgba=np.zeros((32, 64, 4), np.float32), intensity=1.0, rotation=0.0)
        on, off = _gpu(blue_noise, False, sampling=True), _gpu(blue_noise, False, sampling=False)
        con, coff = scenes.apply(on, scene), scenes.apply(off, scene)
        for f in range(6):
            _moving_step([(on, con), (off, coff)], scene, f, w, h)
            for n in CAMERA_BUFFERS:
                assert_bits_equal(on.read_buffer(con, n), off.read_buffer(coff, n), f"{kind} frame {f + 1} {n}")
        if kind == "black":
            assert on.get_stat(STAT_ENVIRONMENT_MAP_DISTRIBUTION_BUILDS) == 1
            assert E.parse_distribution(on.read_scene("environment_map_distribution"))[2] == 0.0
        else:
            assert on.get_stat(STAT_ENVIRONMENT_MAP_DISTRIBUTION_BUILDS) == 0


@pytest.mark.gpu
def test_distribution_life_cycle(blue_noise):
    """Builds and frees follow the rule: the option turning on with a map set builds; a new intensity or rotation alone does not;
    new texels of another size do; the option turning off frees (no distribution to read) and on again rebuilds; clearing the map
    frees; the frames after turning the option off are the option-off frames' in the Reference-free image mode's K13 input."""
    from strolle_b200.engine import StrolleError
    e = _gpu(blue_noise, sampling=False)
    scenes.apply(e, scenes.env_courtyard(64, 36))
    builds = lambda: e.get_stat(STAT_ENVIRONMENT_MAP_DISTRIBUTION_BUILDS)
    e.tick()
    assert builds() == 0
    e.set_option(OPT_ENVIRONMENT_MAP_SAMPLING, 1)
    assert builds() == 0
    e.tick(); assert builds() == 1
    e.tick(); assert builds() == 1
    e.set_environment_map(scenes.courtyard_sky(), 3.0, 1.0); e.tick()
    assert builds() == 1
    e.set_environment_map(MAPS["odd"](), 1.0, 0.0); e.tick()
    assert builds() == 2
    assert E.parse_distribution(e.read_scene("environment_map_distribution"))[:2] == (37, 13)
    e.set_option(OPT_ENVIRONMENT_MAP_SAMPLING, 0); e.tick()
    with pytest.raises(StrolleError):
        e.read_scene("environment_map_distribution")
    e.set_option(OPT_ENVIRONMENT_MAP_SAMPLING, 1); e.tick()
    assert builds() == 3
    e.set_environment_map(None); e.tick()
    with pytest.raises(StrolleError):
        e.read_scene("environment_map_distribution")
    e.set_environment_map(MAPS["odd"](), 1.0, 0.0); e.tick()
    assert builds() == 4


def _devices(n):
    import torch
    have = max(torch.cuda.device_count(), 1)
    return [k % have for k in range(n)]


@pytest.mark.gpu
@pytest.mark.parametrize("n,size", [(2, (320, 288)), (3, (256, 400))])
def test_row_strips_match_single_gpu(blue_noise, n, size):
    """The option on, env_courtyard as n row strips (st_multi_*, which forwards the option to every member): every camera buffer is
    the single-GPU frame's, bit for bit, over 7 moving frames."""
    import strolle_b200
    w, h = size
    scene = _scene("env_courtyard", w, h)
    one = _gpu(blue_noise, False)
    grp = strolle_b200.MultiEngine(_devices(n), blue_noise=blue_noise)
    grp.set_option(OPT_ENVIRONMENT_MAP_SAMPLING, 1)
    c1, cn = scenes.apply(one, scene), scenes.apply(grp, scene)
    for f in range(7):
        _moving_step([(one, c1), (grp, cn)], scene, f, w, h)
        for name in CAMERA_BUFFERS:
            assert_bits_equal(grp.read_buffer(cn, name), one.read_buffer(c1, name), f"{n} strips frame {f + 1} {name}")
    assert grp.peer_errors(cn) == 0


def _frame_stats(blue_noise, name, sampling, frames, w=160, h=90):
    """Mean and per-pixel variance of the composed frame's luminance over `frames` frames, denoising off, camera still."""
    sc = _scene(name, w, h)
    sc["camera"] = dict(sc["camera"], denoise=False)
    e = _gpu(blue_noise, False, sampling=sampling)
    cam = scenes.apply(e, sc)
    acc, acc2 = 0.0, 0.0
    for f in range(frames):
        e.tick(); e.render_camera(cam)
        y = e.read_buffer(cam, "output").reshape(-1, 4)[:, :3].astype(np.float64) @ np.array([0.2126, 0.7152, 0.0722])
        acc, acc2 = acc + y, acc2 + y * y
    mean = acc / frames
    return mean, acc2 / frames - mean * mean


@pytest.mark.gpu
def test_frame_mean_kept_and_variance_lower(blue_noise):
    """256 composed frames with denoising off: on env_courtyard the mean luminance with the option on is within 2% of the option-off
    mean; on env_sunlit the per-pixel variance over frames is lower with it."""
    m_on, _ = _frame_stats(blue_noise, "env_courtyard", True, 256)
    m_off, _ = _frame_stats(blue_noise, "env_courtyard", False, 256)
    rel = abs(m_on.mean() / m_off.mean() - 1.0)
    _, v_on = _frame_stats(blue_noise, "env_sunlit", True, 256)
    _, v_off = _frame_stats(blue_noise, "env_sunlit", False, 256)
    print(f"env_courtyard mean luminance on {m_on.mean():.5g} off {m_off.mean():.5g} (relative {rel:.3g}); "
          f"env_sunlit per-pixel variance on {v_on.mean():.5g} off {v_off.mean():.5g} (factor {v_off.mean() / v_on.mean():.3g})")
    assert rel < 0.02 and v_on.mean() < v_off.mean()
