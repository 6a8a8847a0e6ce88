"""numpy restatement of simulate!(sys, ::MTSIntegrator) and simulate!(sys, ::MTSLangevinIntegrator) (mts_substeps! and the
outer loop, src/simulators.jl:1783-1940) over caller-supplied per-level forces, with the engine's draws
(include/mollyb200.h mb_simulate_mts): xi of atom i (1-based) at innermost substep k (0-based within outer step n) is the
Box-Muller transform of the Philox4x32-10 block with counter (i, n, k, ctr1_lo) and key (key_lo, key_hi). Forces come from
the caller (the C oracle, oracle/bonded.py, oracle/pme.py, oracle/triclinic.py), so the arithmetic is independent of the
engine's. Float64 throughout."""
import math

import numpy as np

import thermostat_oracle as tho


def normals(step, substep, n, rng, sd=1.0):
    """(n, 3) draws sd * xi of atoms 1..n at (outer step, innermost substep); rng = (ctr1_lo, ctr1_hi, key_lo, key_hi)."""
    idx = np.arange(1, n + 1, dtype=np.uint64)
    w = tho.philox4x32_10([idx, np.full(n, step & 0xFFFFFFFF, np.uint64), np.full(n, substep, np.uint64),
                           np.full(n, rng[0], np.uint64)], rng[2], rng[3])
    w = [np.asarray(x, np.float64) for x in w]
    u1, u2 = (w[0] + 1.0) * (1.0 / 4294967296.0), w[1] * (1.0 / 4294967296.0)
    u3, u4 = (w[2] + 1.0) * (1.0 / 4294967296.0), w[3] * (1.0 / 4294967296.0)
    r1, r2 = np.sqrt(-2.0 * np.log(u1)), np.sqrt(-2.0 * np.log(u3))
    two_pi = 6.283185307179586
    sd = np.broadcast_to(np.asarray(sd, np.float64).reshape(-1), (n,))
    return np.stack([sd * r1 * np.cos(two_pi * u2), sd * r1 * np.sin(two_pi * u2), sd * r2 * np.cos(two_pi * u4)], 1)


def coefficients(dt, friction, fractions):
    """MTSLangevinIntegrator's vel_scale and noise_scale (src/simulators.jl:1747-1757)."""
    c = math.exp(-dt * friction / fractions[-1])
    return c, math.sqrt(1 - c * c)


def remove_cm(v, mass):
    m = np.asarray(mass, np.float64)[:, None]
    return v - (m * v).sum(0) / m.sum()


def simulate_mts(level_forces, x, v, mass, dt, n_steps, fractions, wrap, remove_cm_every=1, init_step=0, langevin=None,
                 counts=None):
    """level_forces[l](x) -> forces (n, 3) of level l (fractions[l] = ordered_fractions[l], fractions[0] = 1); wrap(x) ->
    wrapped coordinates. langevin = (kT, friction, rng) for MTSLangevinIntegrator, rng = (ctr1_lo, ctr1_hi, key_lo, key_hi).
    counts: a list that receives the number of evaluations of each level. Returns (x, v) after n_steps outer steps."""
    m = np.asarray(mass, np.float64)[:, None]
    inv_m = np.where(m > 0, 1.0 / np.where(m > 0, m, 1.0), 0.0)  # calc_accels: massless -> 0
    n, n_levels = len(m), len(fractions)
    if langevin is not None:
        kT, friction, rng = langevin
        c, ns = coefficients(dt, friction, fractions)
        sigma = ns * np.sqrt(kT * inv_m[:, 0])
    if counts is not None:
        counts[:] = [0] * n_levels
    st = dict(x=wrap(np.asarray(x, np.float64).copy()), v=np.asarray(v, np.float64).copy(), acc=np.zeros((n, 3)), k=0)
    if init_step == 0 and remove_cm_every != 0:
        st["v"] = remove_cm(st["v"], mass)

    def forces(level):
        if counts is not None:
            counts[level] += 1
        st["acc"] = level_forces[level](st["x"]) * inv_m

    def substeps(level, n_parent, recompute, step):  # mts_substeps!
        n_sub = fractions[level]
        dt_x = dt / n_sub
        dt_v = dt_x / 2
        for _ in range(n_sub // n_parent):
            if recompute:
                forces(level)
            st["v"] = st["v"] + st["acc"] * dt_v
            if level == n_levels - 1:
                if langevin is None:
                    st["x"] = st["x"] + st["v"] * dt_x
                else:
                    st["x"] = st["x"] + st["v"] * (dt_x / 2)
                    st["v"] = c * st["v"] + normals(step, st["k"], n, rng, sigma)
                    st["x"] = st["x"] + st["v"] * (dt_x / 2)
                st["x"] = wrap(st["x"])
                st["k"] += 1
            else:
                substeps(level + 1, n_sub, True, step)
            forces(level)
            st["v"] = st["v"] + st["acc"] * dt_v
            recompute = False

    recompute = True  # the outer level's forces are reused from one outer step to the next
    for step in range(init_step + 1, init_step + n_steps + 1):
        st["k"] = 0
        substeps(0, 1, recompute, step)
        recompute = False
        if remove_cm_every != 0 and step % remove_cm_every == 0:
            st["v"] = remove_cm(st["v"], mass)
    return st["x"], st["v"]
