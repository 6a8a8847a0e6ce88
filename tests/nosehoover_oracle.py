"""numpy restatement of simulate!(sys, ::NoseHoover) (src/simulators.jl:1534-1614). No draws are involved, so the whole
trajectory is pinned. Forces come from the caller (the C oracle, oracle/bonded.py, oracle/pme.py, oracle/triclinic.py),
so the arithmetic is independent of the engine's. Float64 throughout."""
import numpy as np

from langevin_oracle import remove_cm


def zeta_step(zeta, mv2_old, mv2_half, dt, damping, nf_kT):
    """zeta after one step from sum m|v|^2 of the full-step (mv2_old) and half-step (mv2_half) velocities: T / T0 =
    sum m|v|^2 / (Nf k T0) (src/simulators.jl:1575-1579)."""
    coef = dt / (2 * damping * damping)
    zeta_half = zeta + coef * (mv2_old / nf_kT - 1.0)
    return zeta_half + coef * (mv2_half / nf_kT - 1.0)


def simulate_nose_hoover(fe, x, v, mass, dt, n_steps, kT, damping, wrap, remove_cm_every=1, init_step=0):
    """fe(x) -> forces (n, 3); wrap(x) -> wrapped coordinates. Returns (x, v, zeta) after n_steps; zeta starts at 0, as in
    every call of the reference."""
    m = np.asarray(mass, np.float64)[:, None]
    inv_m = np.where(m > 0, 1.0 / np.where(m > 0, m, 1.0), 0.0)
    n = len(m)
    nf_kT = (3 * n - 3) * kT
    x = wrap(np.asarray(x, np.float64).copy())
    v = np.asarray(v, np.float64).copy()
    if init_step == 0 and remove_cm_every != 0:
        v = remove_cm(v, mass)
    a = fe(x) * inv_m
    zeta = 0.0
    for step in range(init_step + 1, init_step + n_steps + 1):
        v_half = v + (a - v * zeta) * (dt / 2)
        x = wrap(x + v_half * dt)
        mv2_old = float((m * v * v).sum())
        mv2_half = float((m * v_half * v_half).sum())
        zeta = zeta_step(zeta, mv2_old, mv2_half, dt, damping, nf_kT)
        a = fe(x) * inv_m
        v = (v_half + a * (dt / 2)) / (1 + zeta * (dt / 2))
        if remove_cm_every != 0 and step % remove_cm_every == 0:
            v = remove_cm(v, mass)
    return x, v, zeta
