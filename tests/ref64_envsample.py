"""ST_OPT_ENVIRONMENT_MAP_SAMPLING restated in numpy (DESIGN.md §2 "Environment map sampling"): the distribution bit for bit in
float32 (np.cumsum over float32 is the sequential running sum the rule names), and the density and K12's mixture density in float64
for quadrature and chi-squared checks."""
import math

import numpy as np


def sin_rows(H):
    """Each row's sin(pi (i + 0.5) / H), in double, rounded to f32."""
    return np.sin(math.pi * (np.arange(H, dtype=np.float64) + 0.5) / H).astype(np.float32)


def weights(texels):
    """The f32 weights: the largest RGB channel over rows i-1..i+1 (clamped) and columns j-1..j+1 (wrapped), times sin_rows."""
    t = np.asarray(texels, np.float32)[..., :3].max(axis=2)
    H = t.shape[0]
    rows = np.maximum(np.maximum(t[np.maximum(np.arange(H) - 1, 0)], t), t[np.minimum(np.arange(H) + 1, H - 1)])
    m = np.maximum(np.maximum(np.roll(rows, 1, axis=1), rows), np.roll(rows, -1, axis=1))
    return (m * sin_rows(H)[:, None]).astype(np.float32)


def cdfs(texels):
    """(marginal CDF [H], conditional CDFs [H, W], total) as the device builds them."""
    cond = np.cumsum(weights(texels), axis=1, dtype=np.float32)
    marg = np.cumsum(cond[:, -1], dtype=np.float32)
    return marg, cond, marg[-1]


def cell_probabilities(marg, cond):
    """Each cell's probability as the draw realises it: (row's marginal difference / total) (cell's conditional difference / row's
    last value), float64."""
    m = np.asarray(marg, np.float64); c = np.asarray(cond, np.float64)
    pr = np.diff(np.concatenate([[0.0], m])) / m[-1]
    rl = c[:, -1:]
    pc = np.diff(np.concatenate([np.zeros((c.shape[0], 1)), c], axis=1), axis=1) / np.where(rl > 0, rl, 1.0)
    return pr[:, None] * pc


def uv64(d, rotation):
    d = np.asarray(d, np.float64)
    theta = np.arccos(np.clip(d[:, 1], -1.0, 1.0))
    phi = np.arctan2(d[:, 0], -d[:, 2])
    return (phi + rotation) / (2.0 * math.pi) + 0.5, theta / math.pi


def env_pdf64(prob, rotation, d):
    """The solid-angle density at directions d (n x 3): the cell's probability times W H / (2 pi^2 sin theta)."""
    H, W = prob.shape
    u, v = uv64(d, rotation)
    j = np.floor(u * W).astype(np.int64) % W
    i = np.clip(np.floor(v * H).astype(np.int64), 0, H - 1)
    st = np.sqrt(np.maximum(0.0, 1.0 - np.asarray(d, np.float64)[:, 1] ** 2))
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(prob[i, j] > 0, prob[i, j] * W * H / (2.0 * math.pi ** 2 * st), 0.0)


def ggx_pdf64(n, v, w, roughness):
    """The solid-angle density of the reference's GGX reflection sampler at w (0 where it cannot reach)."""
    a = min(max(roughness, 0.089 * 0.089), 1.0)
    a2 = a * a
    h = w + v[None, :]
    h = h / np.linalg.norm(h, axis=1, keepdims=True)
    ndh, hdv = np.clip(h @ n, 0.0, 1.0), np.clip(h @ v, 0.0, 1.0)
    dd = (ndh * a2 - ndh) * ndh + 1.0
    D = a2 / (math.pi * dd * dd)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where((ndh > 0) & (hdv > 0), D * ndh / (4.0 * hdv), 0.0)


def mixture64(prob, rotation, n, v, metallic, roughness, w):
    """(q, kappa) of K12's one-sample mixture at directions w."""
    up = (w @ n) > 0
    pg = ggx_pdf64(n, v, w, roughness) if metallic > 0 else np.zeros(len(w))
    m = metallic
    kappa = np.where(up, (1 - m) ** 2 / 2, 0.0) + np.where(pg > 0, m * m, 0.0)
    pb = np.where(up, (1 - m) / (2 * math.pi), 0.0) + m * pg
    return 0.5 * pb + 0.5 * env_pdf64(prob, rotation, w), kappa


def sphere_grid(nu, nv):
    """Midpoint quadrature over the sphere in (u, v) at rotation 0: directions (nu nv x 3), solid-angle weights, cell (u, v)."""
    u = (np.arange(nu) + 0.5) / nu
    v = (np.arange(nv) + 0.5) / nv
    uu, vv = np.meshgrid(u, v)
    theta, phi = vv.ravel() * math.pi, (uu.ravel() - 0.5) * 2.0 * math.pi
    d = np.stack([np.sin(theta) * np.sin(phi), np.cos(theta), -np.sin(theta) * np.cos(phi)], 1)
    dw = np.sin(theta) * (math.pi / nv) * (2.0 * math.pi / nu)
    return d, dw, uu.ravel(), vv.ravel()
