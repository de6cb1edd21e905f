"""Shared helpers for the parity tests: drive the CUDA engine and the CPU oracle with the same
Engine-API calls and compare buffers bit-for-bit (NaN == NaN; the reference itself stores NaN
oct-normals for empty GI reservoirs, strolle-gpu/src/reservoir/gi.rs:47 + normal.rs:10)."""
import numpy as np

CAMERA_BUFFERS = [
    "prim_gbuffer_d0_a", "prim_gbuffer_d0_b", "prim_gbuffer_d1_a", "prim_gbuffer_d1_b", "prim_surface_map_a", "prim_surface_map_b",
    "reprojection_map", "velocity_map", "di_reservoirs_0", "di_reservoirs_1", "di_reservoirs_2", "di_diff_samples", "di_diff_prev_colors",
    "di_diff_curr_colors", "di_diff_moments_a", "di_diff_moments_b", "di_diff_stash", "di_spec_samples", "gi_d0", "gi_d1", "gi_d2",
    "gi_reservoirs_0", "gi_reservoirs_1", "gi_reservoirs_2", "gi_reservoirs_3", "gi_diff_samples", "gi_diff_prev_colors",
    "gi_diff_curr_colors", "gi_diff_moments_a", "gi_diff_moments_b", "gi_diff_stash", "gi_spec_samples", "ref_hits", "ref_rays",
    "ref_colors", "prim_triangle_ids", "output",
]
SCENE_BUFFERS = ["triangles", "bvh", "materials", "lights", "world", "transmittance_lut", "scattering_lut", "sky_lut"]


def bits_equal(a, b):
    """Bit-exact equality of two float32 arrays, treating any NaN as equal to any NaN."""
    a = np.asarray(a, dtype=np.float32).reshape(-1)
    b = np.asarray(b, dtype=np.float32).reshape(-1)
    if a.shape != b.shape:
        return False, f"shape {a.shape} vs {b.shape}"
    ai, bi = a.view(np.uint32), b.view(np.uint32)
    both_nan = np.isnan(a) & np.isnan(b)
    bad = (ai != bi) & ~both_nan
    n = int(bad.sum())
    if n == 0:
        return True, ""
    idx = np.flatnonzero(bad)[:5]
    return False, f"{n}/{a.size} words differ; first at {idx.tolist()}: {a[idx].tolist()} vs {b[idx].tolist()}"


def assert_bits_equal(a, b, what=""):
    ok, msg = bits_equal(a, b)
    assert ok, f"{what}: {msg}"


def rel_l2(a, b):
    a = np.asarray(a, dtype=np.float64).reshape(-1)
    b = np.asarray(b, dtype=np.float64).reshape(-1)
    den = np.sqrt(np.sum(b * b))
    return float(np.sqrt(np.sum((a - b) ** 2)) / den) if den > 0 else float(np.sqrt(np.sum((a - b) ** 2)))


def write_buffer(engine, cam, name, array):
    """Overwrites a per-camera device buffer with `array` (float32 words; uint32 bit patterns are taken as they are), through
    st_buffer_device_ptr and a zero-copy torch view.  The engine is synchronised before and after, so the write lands between
    two `render_range` calls."""
    import torch
    from strolle_b200.multigpu import _DevArray
    ptr, nbytes = engine.buffer_device_ptr(cam, name)
    a = np.ascontiguousarray(np.asarray(array)).reshape(-1).view(np.float32)
    assert a.size * 4 == nbytes, f"{name}: {a.size * 4} bytes for a {nbytes}-byte buffer"
    engine.synchronize()
    torch.as_tensor(_DevArray(ptr, a.size), device="cuda").copy_(torch.from_numpy(a.copy()))
    torch.cuda.synchronize()
    engine.synchronize()


def check_within(got, want, bound, what=""):
    """Per-value comparison with a per-value bound: NaN expected -> NaN, +-inf expected -> the same inf, otherwise
    |got - want| <= bound.  Returns the largest |got - want| / bound over the finite values (0 where both are 0)."""
    got = np.asarray(got, dtype=np.float64)
    want = np.broadcast_to(np.asarray(want, dtype=np.float64), got.shape)
    bound = np.broadcast_to(np.asarray(bound, dtype=np.float64), got.shape)
    nan, inf = np.isnan(want), np.isinf(want)
    bad = (nan & ~np.isnan(got)) | (inf & (got != want))
    fin = ~nan & ~inf
    with np.errstate(invalid="ignore", divide="ignore"):
        err = np.where(fin, np.abs(got - want), 0.0)
        ratio = np.where(err == 0, 0.0, err / bound)
    ratio = np.where(fin & np.isnan(ratio), np.inf, ratio)
    bad |= fin & ~(ratio <= 1.0)
    if bad.any():
        idx = np.flatnonzero(bad.reshape(-1))[:5]
        g, w, b = got.reshape(-1)[idx], want.reshape(-1)[idx], bound.reshape(-1)[idx]
        raise AssertionError(f"{what}: {int(bad.sum())}/{bad.size} values outside the bound; first at flat {idx.tolist()}: "
                             f"got {g.tolist()} want {w.tolist()} bound {b.tolist()}")
    return float(ratio.max()) if ratio.size else 0.0


def primary_rays(scene_camera, engine_like, cam):
    """Camera rays of every pixel as an (n, 8) ray stream, rebuilt from the G-buffer-independent
    camera uniform so that both implementations get identical inputs."""
    raise NotImplementedError


def random_rays(n, seed, lo, hi, max_len=None):
    rng = np.random.RandomState(seed)
    o = rng.uniform(lo, hi, size=(n, 3)).astype(np.float32)
    d = rng.normal(size=(n, 3)).astype(np.float32)
    d /= np.linalg.norm(d, axis=1, keepdims=True).astype(np.float32)
    rays = np.zeros((n, 8), dtype=np.float32)
    rays[:, 0:3] = o
    rays[:, 4:7] = d
    rays[:, 3] = np.float32(3.4028234663852886e38) if max_len is None else rng.uniform(0.1, max_len, size=n).astype(np.float32)
    return rays
