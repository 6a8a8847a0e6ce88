"""numpy restatement of simulate!(sys, ::LangevinSplitting) (src/simulators.jl:1252-1398), force-recompute rule included,
with the engine's draws (include/mollyb200.h mb_simulate_langevin_splitting): xi of atom i (1-based) at the j-th O of step
n is langevin_oracle.normals(n, ...) with ctr1 + j (the reference advances one ctr1 by one per O over the whole run; the two
agree in distribution only). Forces come from the caller (the C oracle, oracle/bonded.py,
oracle/pme.py, oracle/triclinic.py), so the arithmetic is independent of the engine's. Float64 throughout."""
import re

import numpy as np

import langevin_oracle as lo


def force_computation_steps(splitting):
    """The reference's force_computation_steps: per letter, whether that B recomputes the forces."""
    known = re.search(r"^.*B[^B]*A[^B]*$", splitting) is None
    out = []
    for op in splitting:
        if op == "A":
            known = False
        if op == "B" and not known:
            known = True
            out.append(True)
        else:
            out.append(False)
    return out


def evaluations_per_step(splitting):
    return sum(force_computation_steps(splitting))


def simulate_splitting(fe, x, v, mass, dt, n_steps, kT, friction, splitting, rng, wrap, remove_cm_every=1, init_step=0,
                       count=None):
    """fe(x) -> forces (n, 3); wrap(x) -> wrapped coordinates; rng = (ctr1_lo, ctr1_hi, key_lo, key_hi). Returns (x, v) after
    n_steps. count: a list that receives the number of force evaluations of each step (the initial one excluded)."""
    if not all(op in "ABO" for op in splitting):
        raise ValueError("splitting must contain only A, B, and O steps")
    m = np.asarray(mass, np.float64)[:, None]
    inv_m = np.where(m > 0, 1.0 / np.where(m > 0, m, 1.0), 0.0)
    n = len(m)
    n_o = splitting.count("O")
    if n_o > 0:
        vel_scales = np.exp((-friction * dt / n_o) * inv_m)
        noise_scales = np.sqrt(kT * inv_m * (1.0 - vel_scales ** 2))
    ctr1 = rng[0] | (rng[1] << 32)
    x = wrap(np.asarray(x, np.float64).copy())
    v = np.asarray(v, np.float64).copy()
    if init_step == 0 and remove_cm_every != 0:
        v = lo.remove_cm(v, mass)
    f = fe(x)
    eff = [dt / splitting.count(op) for op in splitting]
    recompute = force_computation_steps(splitting)
    for step in range(init_step + 1, init_step + n_steps + 1):
        c1 = ctr1
        evals = 0
        for j, op in enumerate(splitting):
            if op == "A":
                x = wrap(x + v * eff[j])
            elif op == "B":
                if recompute[j]:
                    f = fe(x)
                    evals += 1
                v = v + eff[j] * (f * inv_m)
            else:
                c = c1 % 2 ** 64
                v = vel_scales * v + lo.normals(step, n, (c & 0xFFFFFFFF, c >> 32, rng[2], rng[3]), noise_scales[:, 0])
                c1 += 1
        x = wrap(x)
        if remove_cm_every != 0 and step % remove_cm_every == 0:
            v = lo.remove_cm(v, mass)
        if count is not None:
            count.append(evals)
    return x, v
