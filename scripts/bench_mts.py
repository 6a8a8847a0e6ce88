#!/usr/bin/env python
"""Cost and stability of the multiple-time-step integrators on the C3 workload of bench.py (6mrr, 15 954 atoms, f32, device
state, uncoupled).

Compared: VelocityVerlet at 0.5 fs (what C3 runs at: the bond vibrations set the step), MTSIntegrator at a 1 fs outer step
with the bonds and angles substepped twice (si_fractions (2, 2, 1) for bonds, angles, torsions), MTSIntegrator at a 2 fs outer
step with si_fractions (4, 4, 2), and MTSLangevinIntegrator (300 K, friction 1 ps^-1) at both configurations. For each:
outer steps/s (median of alternating rounds), ns/day, pair-kernel launches per simulated ps (the engine's force-evaluation
counter over the timed window), and, over a window of `--drift-ps` ps logged every 10 outer steps, the total energy at its
start and end, the least-squares slope of the total energy over the second half of the window (kJ/mol per ns; for the
Langevin runs not a conservation measure) and the mean temperature over that half. The card name and power limit are read
in the same run.

    python scripts/bench_mts.py [--steps 2000] [--rounds 3] [--drift-ps 5]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "tests"), ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)

import bench  # noqa: E402  (workload definitions)
import mbhelpers as H  # noqa: E402

# name -> (outer dt in ps, si_fractions or None for VelocityVerlet, Langevin)
MODES = {"vv-0.5fs": (0.0005, None, False), "mts-1fs(2,2,1)": (0.001, (2, 2, 1), False),
         "mts-2fs(4,4,2)": (0.002, (4, 4, 2), False), "mtsl-1fs(2,2,1)": (0.001, (2, 2, 1), True),
         "mtsl-2fs(4,4,2)": (0.002, (4, 4, 2), True)}


def system(loggers=None):
    import torch
    import mollyb200 as mb
    dtype = np.float32
    sd, inters, _, _, rc, label = bench.workload("c3", dtype)
    atoms = mb.atoms_from_arrays(sd["mass"], sd["charge"], sd["sigma"], sd["eps"], dtype)
    nf = mb.GPUNeighborFinder(dist_cutoff=bench.default_r_list("c3", rc), excluded_pairs=sd["excluded"] + 1,
                              special_pairs=sd["special"] + 1)
    return mb.System(atoms=atoms, coords=torch.from_numpy(sd["coords"]).cuda().contiguous(), boundary=mb.CubicBoundary(*sd["box"]),
                     velocities=torch.from_numpy(sd["velocities"]).cuda().contiguous(), pairwise_inters=inters, neighbor_finder=nf,
                     dtype=dtype, specific_inter_lists=H.sixmrr_specific_lists(sd["golden"]), loggers=loggers), label


def simulator(mode):
    import mollyb200 as mb
    dt, si, lang = MODES[mode]
    if si is None:
        return mb.VelocityVerlet(dt=dt)
    pi = (1, 1)
    if lang:
        return mb.MTSLangevinIntegrator(dt, 300.0, 1.0, pi_fractions=pi, si_fractions=si)
    return mb.MTSIntegrator(dt, pi_fractions=pi, si_fractions=si)


def timed(mode, steps, warmup):
    import mollyb200 as mb
    s, label = system()
    sim = simulator(mode)
    rng = np.random.default_rng(1)
    mb.simulate(s, sim, warmup, rng=rng)
    ev0 = s.stats()["n_force_evals"]
    t0 = time.perf_counter()
    mb.simulate(s, sim, steps, init_step=warmup, rng=rng)  # the call ends in a device synchronise
    rate = steps / (time.perf_counter() - t0)
    st = s.stats()
    s.close()
    return rate, (st["n_force_evals"] - ev0 - 1) / (steps * sim.dt), st["graph_mode"], label


def drift(mode, ps):
    import mollyb200 as mb
    s, _ = system({"e": mb.TotalEnergyLogger(10), "t": mb.TemperatureLogger(10)})
    sim = simulator(mode)
    n = int(round(ps / sim.dt))
    mb.simulate(s, sim, n, rng=np.random.default_rng(2))
    e = np.array([float(v) for v in mb.values(s.loggers["e"])])
    temp = np.array([float(v) for v in mb.values(s.loggers["t"])])
    s.close()
    t = np.arange(len(e)) * 10 * sim.dt  # ps
    h = len(e) // 2
    if not np.all(np.isfinite(e)):
        return None, e[0], e[-1], float("nan")
    return np.polyfit(t[h:], e[h:], 1)[0] * 1000.0, e[0], e[-1], temp[h:].mean()  # kJ/mol per ns


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--warmup", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--drift-ps", type=float, default=5.0)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()
    print(f"card: {card[0] if card else 'unknown'}")
    rates = {m: [] for m in MODES}
    info = {}
    for _ in range(args.rounds):
        for m in MODES:
            r, pairs_per_ps, graph, label = timed(m, args.steps, args.warmup)
            rates[m].append(r)
            info[m] = (pairs_per_ps, graph)
    print(f"c3: {label}, {args.steps} timed outer steps, {args.rounds} alternating rounds; drift over {args.drift_ps} ps")
    for m in MODES:
        dt = MODES[m][0]
        med = np.median(rates[m])
        slope, e0, e1, tm = drift(m, args.drift_ps)
        d = "NaN" if slope is None else f"{slope:+9.1f} kJ/mol/ns"
        print(f"  {m:16s} steps/s {med:8.1f} (range {min(rates[m]):8.1f} - {max(rates[m]):8.1f})  ns/day {med * dt * 86.4:7.2f}  "
              f"pair launches/ps {info[m][0]:7.1f}  graph {info[m][1]}  E slope (2nd half) {d}  E {e0:.1f} -> {e1:.1f}  "
              f"<T> (2nd half) {tm:.1f} K")


if __name__ == "__main__":
    main()
