"""numpy restatements of simulate!(sys, ::Verlet), simulate!(sys, ::StormerVerlet) and simulate!(sys, ::OverdampedLangevin)
(src/simulators.jl:868-955, :970-1063, :1427-1490), written as the reference loops are. StormerVerlet keeps coords_last
as the reference does; OverdampedLangevin takes the engine's draws (langevin_oracle.normals, include/mollyb200.h
mb_simulate_overdamped_langevin). Forces come from the caller, so the arithmetic is independent of the engine's. Float64
throughout."""
import numpy as np

from langevin_oracle import normals, remove_cm


def _inv_mass(mass):
    m = np.asarray(mass, np.float64)[:, None]
    return np.where(m > 0, 1.0 / np.where(m > 0, m, 1.0), 0.0)


def simulate_verlet(fe, x, v, mass, dt, n_steps, wrap, remove_cm_every=1, init_step=0):
    """fe(x) -> forces (n, 3); wrap(x) -> wrapped coordinates. Returns (x, v) after n_steps."""
    inv_m = _inv_mass(mass)
    x = wrap(np.asarray(x, np.float64).copy())
    v = np.asarray(v, np.float64).copy()
    if init_step == 0 and remove_cm_every != 0:
        v = remove_cm(v, mass)
    for step in range(init_step + 1, init_step + n_steps + 1):
        a = fe(x) * inv_m
        v = v + a * dt
        x = x + v * dt
        x = wrap(x)
        if remove_cm_every != 0 and step % remove_cm_every == 0:
            v = remove_cm(v, mass)
    return x, v


def simulate_stormer_verlet(fe, x, v, mass, dt, n_steps, wrap, vector, init_step=0):
    """vector(a, b) -> the minimum-image displacement b - a (the boundary's `vector`). Returns (x, v) after n_steps."""
    inv_m = _inv_mass(mass)
    x = wrap(np.asarray(x, np.float64).copy())
    v = np.asarray(v, np.float64).copy()
    coords_last = np.zeros_like(x)
    dt_sq = dt * dt
    for step in range(init_step + 1, init_step + n_steps + 1):
        a = fe(x) * inv_m
        coords_copy = x.copy()
        if step == init_step + 1:
            x = x + v * dt + (a * dt_sq) / 2
        else:
            x = x + vector(coords_last, x) + a * dt_sq
        x = wrap(x)
        v = vector(coords_copy, x) / dt
        coords_last = coords_copy
    return x, v


def simulate_overdamped(fe, x, v, mass, dt, n_steps, kT, friction, rng, wrap, remove_cm_every=1, init_step=0):
    """rng = (ctr1_lo, ctr1_hi, key_lo, key_hi). Returns (x, v) after n_steps."""
    inv_m = _inv_mass(mass)
    n = len(inv_m)
    x = wrap(np.asarray(x, np.float64).copy())
    v = np.asarray(v, np.float64).copy()
    if init_step == 0 and remove_cm_every != 0:
        v = remove_cm(v, mass)
    noise_prefac = np.sqrt((2 / friction) * dt)
    for step in range(init_step + 1, init_step + n_steps + 1):
        a = fe(x) * inv_m
        noise = normals(step, n, rng, np.sqrt(kT * inv_m[:, 0]))  # random_velocities!: sqrt(kT / m) xi
        x = x + (a / friction) * dt + noise_prefac * noise
        x = wrap(x)
        if remove_cm_every != 0 and step % remove_cm_every == 0:
            v = remove_cm(v, mass)
    return x, v


def simulate_velocity_verlet(fe, x, v, mass, dt, n_steps, wrap, remove_cm_every=0, init_step=0):
    """simulate!(sys, ::VelocityVerlet) (src/simulators.jl:547-668), for the identities and the reference's protocol."""
    inv_m = _inv_mass(mass)
    x = wrap(np.asarray(x, np.float64).copy())
    v = np.asarray(v, np.float64).copy()
    if init_step == 0 and remove_cm_every != 0:
        v = remove_cm(v, mass)
    a = fe(x) * inv_m
    for step in range(init_step + 1, init_step + n_steps + 1):
        x = wrap(x + v * dt + a * (dt * dt / 2))
        a_new = fe(x) * inv_m
        v = v + (a + a_new) * (dt / 2)
        a = a_new
        if remove_cm_every != 0 and step % remove_cm_every == 0:
            v = remove_cm(v, mass)
    return x, v
