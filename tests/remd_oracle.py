"""numpy restatement of temperature replica exchange: simulate_remd! and remd_exchange! (src/simulators.jl:1965-2206) with
the draw order mollyb200.simulate_remd documents. The integrator of each state is a callable, so the existing integrator
oracles (langevin_oracle.simulate_langevin, nosehoover_oracle.simulate_nose_hoover,
thermostat_oracle.simulate_vv_coupled) compose with the exchange logic here."""
import math

import numpy as np


def simulate_remd(xs, vs, betas, state_indices, integrate, energy, n_steps, dt, exchange_time, init_step, rng, dtype,
                  draws=True):
    """xs, vs: per physical replica (n, 3) arrays, updated in place. integrate(s, x, v, n, start, keys) -> (x, v) runs
    state s's integrator for n steps from step `start`; keys = (rng_ctr1, rng_key), the two draws simulate makes (None
    when draws is False). energy(x) -> U. Returns the state indices, the exchange log and the list of calls
    (replica, state, n, start)."""
    R = len(xs)
    si = list(state_indices)
    n_cycles = int((n_steps * dt) // exchange_time)
    cycle_length = n_steps // n_cycles if n_cycles > 0 else 0
    remaining = n_steps % n_cycles if n_cycles > 0 else n_steps
    log = dict(indices=[], steps=[], deltas=[], n_attempts=0)
    calls = []

    def run(length, start):
        for i in range(R):
            keys = (int(rng.integers(0, 2 ** 63)), int(rng.integers(0, 2 ** 63))) if draws else None
            x, v = integrate(si[i], xs[i], vs[i], length, start, keys)
            xs[i][...] = np.asarray(x).astype(dtype)
            vs[i][...] = np.asarray(v).astype(dtype)
            calls.append((i, si[i], length, start))

    for cycle in range(1, n_cycles + 1):
        run(cycle_length, init_step + (cycle - 1) * cycle_length)
        for i in range(cycle % 2, R - 1, 2):
            j = i + 1
            log["n_attempts"] += 1
            m, n = si[i], si[j]
            bm, bn = betas[m], betas[n]
            delta = (bn - bm) * (float(energy(xs[i])) - float(energy(xs[j])))
            if delta <= 0 or rng.random() < math.exp(-delta):
                si[i], si[j] = n, m
                if bm != bn:
                    vs[i] *= np.asarray(math.sqrt(bm / bn), dtype)
                    vs[j] *= np.asarray(math.sqrt(bn / bm), dtype)
                log["indices"].append((i, j))
                log["steps"].append(init_step + cycle * cycle_length)
                log["deltas"].append(delta)
    if remaining > 0:
        run(remaining, init_step + n_cycles * cycle_length)
    log["end_step"] = init_step + n_steps
    return si, log, calls
