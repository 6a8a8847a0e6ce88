"""numpy (f64) restatement of DPDInteraction (src/interactions/dpd.jl:57-142) and of the DPDVelocityVerlet loop
(src/simulators.jl:711-842) as the engine runs them (csrc/dpd.cuh, include/mollyb200.h mb_set_dpd / mb_simulate_dpd_vv):
the pairwise draw with the numpy Philox of thermostat_oracle, the pair term in the engine's order of operations, minimum
image in cubic or triclinic boxes, exclusions, harmonic bonds, the CM-removal schedule and each call's F0 with v(t)."""
import math

import numpy as np

import thermostat_oracle as tho

_M32 = 0xFFFFFFFF


def normal(i, j, step, key):
    """xi_ij of `step` for 0-based indices (arrays or scalars): counter (min + 1, max + 1, step_lo, step_hi), key
    (key_lo, key_hi), Box-Muller of words 0 and 1 with the C library's log and cos."""
    i, j = np.asarray(i, np.int64), np.asarray(j, np.int64)
    lo, hi = np.minimum(i, j) + 1, np.maximum(i, j) + 1
    step = int(step)
    w = tho.philox4x32_10([lo.astype(np.uint64), hi.astype(np.uint64), np.full(lo.shape, step & _M32, np.uint64),
                           np.full(lo.shape, (step >> 32) & _M32, np.uint64)], key & _M32, (key >> 32) & _M32)
    w0, w1 = np.atleast_1d(w[0]), np.atleast_1d(w[1])
    out = np.array([tho.normal(int(a), int(b)) for a, b in zip(w0, w1)], np.float64)
    return out if lo.ndim else float(out[0])


def pair(p, r, d, dv, xi):
    """fr (force on i = fr d, d = c_i - c_j, dv = v_i - v_j) and the energy of pairs at distance r, in the engine's order
    of operations (dpd_pair). p: dict a, gamma, sigma, r_c, dt."""
    r, d, dv, xi = (np.asarray(a, np.float64) for a in (r, d, dv, xi))
    inside = (r < p["r_c"]) & (r != 0)
    rs = np.where(inside, r, 1.0)
    w = 1.0 - rs / p["r_c"]
    inv_r = 1.0 / rs
    f_c = p["a"] * w * inv_r
    rdotv = -(d[..., 0] * dv[..., 0] + d[..., 1] * dv[..., 1] + d[..., 2] * dv[..., 2]) * inv_r * inv_r
    f_d = p["gamma"] * (w * w) * rdotv
    f_r = p["sigma"] * w * xi * (1.0 / math.sqrt(p["dt"])) * inv_r
    e_pre = (p["a"] / 2) * p["r_c"]
    return np.where(inside, f_c + f_d + f_r, 0.0), np.where(inside, e_pre * w * w, 0.0)


def min_image(box):
    """vector(c_i, c_j) = c_j - c_i, minimum image; box: 3 side lengths or a 3 x 3 lower-triangular basis (rows)."""
    b = np.asarray(box, np.float64)
    if b.ndim == 1:
        return lambda a, c: (c - a) - b * np.round((c - a) / b)

    def tric(a, c):  # the basis is lower triangular: reduce z, then y, then x, then search the 27 neighbouring images
        d = c - a
        for k in (2, 1, 0):
            d = d - np.round(d[..., k:k + 1] / b[k, k]) * b[k]
        best = d.copy()
        for sx in (-1, 0, 1):
            for sy in (-1, 0, 1):
                for sz in (-1, 0, 1):
                    e = d + sx * b[0] + sy * b[1] + sz * b[2]
                    better = (e * e).sum(-1) < (best * best).sum(-1)
                    best[better] = e[better]
        return best
    return tric


def pairs_within(x, box, r_c):
    """(i, j, dr) for i < j with |dr| < r_c (dr = c_j - c_i, minimum image), all pairs in order."""
    n = len(x)
    vec = min_image(box)
    b = np.asarray(box, np.float64)
    if b.ndim == 1 and n > 2000:  # candidates from a periodic k-d tree, exact distances below
        from scipy.spatial import cKDTree
        y = np.mod(x, b)
        y[y >= b] = 0.0
        pr = cKDTree(y, boxsize=b).query_pairs(r_c * 1.001, output_type="ndarray")
        pr = np.sort(pr, axis=1)
        pr = pr[np.lexsort((pr[:, 1], pr[:, 0]))]
        ii, jj = pr[:, 0], pr[:, 1]
    else:
        ii, jj = np.triu_indices(n, 1)
    dr = vec(x[ii], x[jj])
    r2 = (dr * dr).sum(-1)
    keep = r2 < r_c * r_c * (1 + 1e-9)
    return ii[keep], jj[keep], dr[keep]


def forces(x, v, box, p, step, excluded=(), bonds=None):
    """Forces (n x 3) and energy of the DPD term (+ harmonic bonds: rows (i, j, k, r0), 0-based) at `step` with velocities
    v. excluded: a set of 0-based (i, j) pairs, i < j, skipped (use_neighbors)."""
    x, v = np.asarray(x, np.float64), np.asarray(v, np.float64)
    f = np.zeros_like(x)
    ii, jj, dr = pairs_within(x, box, p["r_c"])
    if len(excluded):
        keep = np.array([(int(a), int(b)) not in excluded for a, b in zip(ii, jj)], bool)
        ii, jj, dr = ii[keep], jj[keep], dr[keep]
    d = -dr
    r = np.sqrt(d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2])
    xi = normal(ii, jj, step, p["key"]) if len(ii) else np.zeros(0)
    fr, e = pair(p, r, d, v[ii] - v[jj], xi)
    fi = fr[:, None] * d
    np.add.at(f, ii, fi)
    np.add.at(f, jj, -fi)
    energy = float(e.sum())
    if bonds is not None and len(bonds):
        bi, bj = bonds[:, 0].astype(int), bonds[:, 1].astype(int)
        k, r0 = bonds[:, 2], bonds[:, 3]
        ab = min_image(box)(x[bi], x[bj])
        rb = np.sqrt((ab * ab).sum(-1))
        fb = (k * (rb - r0) / rb)[:, None] * ab
        np.add.at(f, bi, fb)
        np.add.at(f, bj, -fb)
        energy += float((0.5 * k * (rb - r0) ** 2).sum())
    return f, energy


def wrap(x, box):
    b = np.asarray(box, np.float64)
    if b.ndim == 1:
        return x - np.floor(x / b) * b
    y = x.copy()
    for k in (2, 1, 0):
        y = y - np.floor(y[..., k:k + 1] / b[k, k]) * b[k]
    return y


def remove_cm(v, mass):
    m = np.asarray(mass, np.float64)[:, None]
    return v - (m * v).sum(0) / m.sum()


def simulate_dpd_vv(x, v, mass, box, p, dt, lam, n_steps, remove_cm_every=1, init_step=0, excluded=(), bonds=None,
                    record=None):
    """One simulate! call of DPDVelocityVerlet (src/simulators.jl:711-842): wrap, CM removal when init_step == 0, F0 at
    init_step with v(t), then n_steps of kick / drift / wrap / v_pred / F(x, v_pred, step) / kick / CM removal.
    record(step, x, v, pe): called after every step (and at init_step) with the state the loggers see."""
    m = np.asarray(mass, np.float64)[:, None]
    x = wrap(np.asarray(x, np.float64), box)
    v = np.asarray(v, np.float64).copy()
    if init_step == 0 and remove_cm_every:
        v = remove_cm(v, mass)
    f, pe = forces(x, v, box, p, init_step, excluded, bonds)
    if record:
        record(init_step, x, v, pe)
    a = f / m
    for step in range(init_step + 1, init_step + n_steps + 1):
        v = v + a * (dt / 2)
        x = wrap(x + v * dt, box)
        v_half = v
        v_pred = v_half + a * ((lam - 0.5) * dt)
        f, pe = forces(x, v_pred, box, p, step, excluded, bonds)
        a = f / m
        v = v_half + a * (dt / 2)
        if remove_cm_every and step % remove_cm_every == 0:
            v = remove_cm(v, mass)
        if record:
            record(step, x, v, pe)
    return x, v
