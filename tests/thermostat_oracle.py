"""numpy restatement of the velocity-rescaling thermostats as the engine runs them (csrc/vrescale.cuh, include/mollyb200.h
mb_set_velocity_coupling): Philox4x32-10 blocks, Box-Muller normals, the Marsaglia-Tsang chi^2 draw, lambda of
ImmediateThermostat / BerendsenThermostat / VelocityRescaleThermostat (src/coupling.jl:82-168, :227-238), and the
reference's VelocityVerlet loop with coupling (src/simulators.jl:547-668) over the C oracle's forces."""
import math

import numpy as np

IMMEDIATE, BERENDSEN, VRESCALE = 1, 2, 3
MAX_PROPOSALS = 64
_M32 = 0xFFFFFFFF


def rng_words(ctr1: int, key: int):
    """(ctr1_lo, ctr1_hi, key_lo, key_hi): what the device reads from the call's rng_ctr1 / rng_key."""
    return (ctr1 & _M32, (ctr1 >> 32) & _M32, key & _M32, (key >> 32) & _M32)


def philox4x32_10(c, k0, k1):
    """Vectorised Philox4x32-10 (Salmon et al. 2011): c is a (4, m) uint64 array of 32-bit words, keys broadcast."""
    c = [np.asarray(x, np.uint64) & _M32 for x in c]
    k0, k1 = np.asarray(k0, np.uint64) & _M32, np.asarray(k1, np.uint64) & _M32
    M0, M1, W0, W1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57), np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)
    m32 = np.uint64(_M32)
    for _ in range(10):
        p0, p1 = M0 * c[0], M1 * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & m32, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & m32]
        k0, k1 = (k0 + W0) & m32, (k1 + W1) & m32
    return c


def block(j, step, rng):
    """Block j of the draws at `step`: counter (0xFFFFFFFF - j, step, ctr1_lo, ctr1_hi), key (key_lo, key_hi)."""
    w = philox4x32_10([_M32 - np.asarray(j, np.uint64), np.asarray(step, np.uint64) & _M32, rng[0], rng[1]], rng[2], rng[3])
    return [int(x) if np.ndim(x) == 0 else x for x in w]


def normal(a, b):
    u1 = (float(a) + 1.0) * (1.0 / 4294967296.0)
    u2 = float(b) * (1.0 / 4294967296.0)
    return math.sqrt(-2.0 * math.log(u1)) * math.cos(6.283185307179586 * u2)


def chi2(k: int, step: int, rng) -> float:
    """2 Gamma(k/2) by Marsaglia-Tsang, proposals from blocks 1, 2, ...; shape < 1: times U^(1/shape), U from block 0."""
    if k <= 0:
        return 0.0
    a = 0.5 * k
    boost = a < 1.0
    d = (a + 1.0 if boost else a) - 1.0 / 3.0
    c = 1.0 / math.sqrt(9.0 * d)
    g = d
    for j in range(1, MAX_PROPOSALS + 1):
        w = block(j, step, rng)
        x = normal(w[0], w[1])
        t = 1.0 + c * x
        if t <= 0.0:
            continue
        v = t * t * t
        u = (w[2] + 1.0) * (1.0 / 4294967296.0)
        if math.log(u) < 0.5 * x * x + d - d * v + d * math.log(v):
            g = d * v
            break
    if boost:
        g *= ((block(0, step, rng)[2] + 1.0) * (1.0 / 4294967296.0)) ** (1.0 / a)
    return 2.0 * g


def lam(kind, K, nf, kT, dt, tau=0.0, n_steps=1, step=0, rng=(0, 0, 0, 0)) -> float:
    """The factor every velocity is scaled by after the step's CM removal; K <= 0 or nf <= 0: 1."""
    if not K > 0 or nf <= 0:
        return 1.0
    t_ratio = kT / (2.0 * K / nf)  # T0 / T
    if kind == IMMEDIATE:
        return math.sqrt(t_ratio)
    if kind == BERENDSEN:
        return math.sqrt(1.0 + (dt / tau) * (t_ratio - 1.0))
    if step % n_steps != 0:
        return 1.0
    c = math.exp(-(dt * n_steps) / tau)
    A = (nf * kT / 2.0) / (nf * K)
    w = block(0, step, rng)
    R = normal(w[0], w[1])
    S = chi2(nf - 1, step, rng)
    lam2 = c + (1.0 - c) * A * (R * R + S) + 2.0 * math.sqrt(c * (1.0 - c) * A) * R
    return math.sqrt(max(lam2, np.finfo(np.float64).eps))


def kind_of(thermostat):
    name = type(thermostat).__name__
    return {"ImmediateThermostat": IMMEDIATE, "BerendsenThermostat": BERENDSEN, "VelocityRescaleThermostat": VRESCALE}[name]


def simulate_vv_coupled(orc, x, v, mass, box, dt, n_steps, thermostat, k, rng, remove_cm_every=1, init_step=0):
    """simulate!(sys, VelocityVerlet(dt, (thermostat,), remove_cm_every), n_steps) in f64 with the oracle's all-pairs forces:
    kick, drift, wrap, forces, kick, CM removal, coupling (src/simulators.jl:616-643). Returns (x, v)."""
    kind = kind_of(thermostat)
    kT = k * thermostat.temperature
    tau = getattr(thermostat, "coupling_const", 0.0)
    every = getattr(thermostat, "n_steps", 1)
    m = np.asarray(mass, np.float64)[:, None]
    nf = 3 * len(m) - 3
    x = np.asarray(x, np.float64).copy()
    x -= np.floor(x / box) * box
    v = np.asarray(v, np.float64).copy()
    if init_step == 0 and remove_cm_every != 0:
        v = orc.remove_cm(v)
    f = orc.forces_allpairs(x, energy=False)[0]
    for step in range(init_step + 1, init_step + n_steps + 1):
        v = v + f / m * (dt / 2)
        x = x + v * dt
        x -= np.floor(x / box) * box
        f = orc.forces_allpairs(x, energy=False)[0]
        v = v + f / m * (dt / 2)
        if remove_cm_every != 0 and step % remove_cm_every == 0:
            v = orc.remove_cm(v)
        K = 0.5 * float(np.sum(m * v * v))
        v = v * lam(kind, K, nf, kT, dt, tau, every, step, rng)
    return x, v
