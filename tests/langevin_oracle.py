"""numpy restatement of simulate!(sys, ::Langevin) (src/simulators.jl:1099-1210, O step src/kernels.jl:723-756) with the
engine's draws (include/mollyb200.h mb_simulate_langevin): xi of atom i (1-based) at step n is the Box-Muller transform of
the Philox4x32-10 block with counter (i, n, ctr1_lo, ctr1_hi) and key (key_lo, key_hi). Forces come from the caller (the C
oracle, oracle/bonded.py, oracle/triclinic.py), so the arithmetic is independent of the engine's. Float64 throughout."""
import math

import numpy as np

import thermostat_oracle as tho


def normals(step, n, rng, sd=1.0):
    """(n, 3) draws sd * xi of atoms 1..n at `step`; rng = (ctr1_lo, ctr1_hi, key_lo, key_hi)."""
    idx = np.arange(1, n + 1, dtype=np.uint64)
    w = tho.philox4x32_10([idx, np.full(n, step & 0xFFFFFFFF, np.uint64), np.full(n, rng[0], np.uint64),
                           np.full(n, rng[1], np.uint64)], rng[2], rng[3])
    w = [np.asarray(x, np.float64) for x in w]
    u1, u2 = (w[0] + 1.0) * (1.0 / 4294967296.0), w[1] * (1.0 / 4294967296.0)
    u3, u4 = (w[2] + 1.0) * (1.0 / 4294967296.0), w[3] * (1.0 / 4294967296.0)
    r1, r2 = np.sqrt(-2.0 * np.log(u1)), np.sqrt(-2.0 * np.log(u3))
    two_pi = 6.283185307179586
    sd = np.broadcast_to(np.asarray(sd, np.float64).reshape(-1), (n,))
    return np.stack([sd * r1 * np.cos(two_pi * u2), sd * r1 * np.sin(two_pi * u2), sd * r2 * np.cos(two_pi * u4)], 1)


def coefficients(dt, friction):
    """Langevin's vel_scale and noise_scale (src/simulators.jl:1092-1097)."""
    c = math.exp(-dt * friction)
    return c, math.sqrt(1 - c * c)


def remove_cm(v, mass):
    m = np.asarray(mass, np.float64)[:, None]
    return v - (m * v).sum(0) / m.sum()


def simulate_langevin(fe, x, v, mass, dt, n_steps, kT, friction, rng, wrap, remove_cm_every=1, init_step=0):
    """fe(x) -> forces (n, 3); wrap(x) -> wrapped coordinates. Returns (x, v) after n_steps."""
    m = np.asarray(mass, np.float64)[:, None]
    inv_m = np.where(m > 0, 1.0 / np.where(m > 0, m, 1.0), 0.0)
    c, ns = coefficients(dt, friction)
    sigma = ns * np.sqrt(kT * inv_m[:, 0])
    n = len(m)
    x = wrap(np.asarray(x, np.float64).copy())
    v = np.asarray(v, np.float64).copy()
    if init_step == 0 and remove_cm_every != 0:
        v = remove_cm(v, mass)
    f = fe(x)
    for step in range(init_step + 1, init_step + n_steps + 1):
        v = v + f * inv_m * dt
        x = x + v * (dt / 2)
        v = c * v + normals(step, n, rng, sigma)
        x = x + v * (dt / 2)
        x = wrap(x)
        if remove_cm_every != 0 and step % remove_cm_every == 0:
            v = remove_cm(v, mass)
        f = fe(x)
    return x, v
