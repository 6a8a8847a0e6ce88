#!/usr/bin/env python
"""Cost of Verlet, StormerVerlet and OverdampedLangevin next to VelocityVerlet, on the C2 and C3 workloads of bench.py (f32,
device state), and of the Andersen thermostat with Verlet and with VelocityVerlet.

The same number of steps with each integrator, alternated over several rounds; the median of the rounds is reported.
OverdampedLangevin runs at the temperature the workload starts at (C2: 90 K, C3: 300 K) with a friction that keeps
Euler-Maruyama stable on the workload's stiffest term (C2: 10 ps^-1, the reference's test value; C3: 1000 ps^-1 for the
bonds to hydrogen). The Andersen thermostat targets that temperature with a 1 ps coupling constant, as C3 of bench.py
does; with VelocityVerlet it is folded into the next step's drift kernel, with Verlet it is a kernel launch of its own after
the step. Prints steps/s and the rebuilds of the timed window for each, with the card name and power limit read in
the same run. The step rate also moves with the rebuild count, which each integrator's trajectory sets, so a second,
profiled window of 200 steps (stream path, CUDA events around each launch) gives the time of the integration kernels alone
per step: K1 + K2 for VelocityVerlet, the one step kernel for the others (the standalone Andersen kernel is not in it).

    python scripts/bench_verlet.py [--steps 1000] [--rounds 3] [--workloads c2,c3]
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

MODES = ("vv", "verlet", "stormer", "overdamped", "vv-andersen", "verlet-andersen")
PROF_STEPS = 200


TEMPERATURE = {"c2": 90.0, "c3": 300.0}  # K: what tests/mbhelpers.lj_fluid and the 6mrr velocities are drawn at


FRICTION = {"c2": 10.0, "c3": 1000.0}  # ps^-1 (OverdampedLangevin)


def simulator(mode, dt, wl):
    import mollyb200 as mb
    andersen = mb.AndersenThermostat(TEMPERATURE[wl], 1.0) if mode.endswith("-andersen") else None
    if mode.startswith("verlet"):
        return mb.Verlet(dt=dt, coupling=andersen)
    if mode == "stormer":
        return mb.StormerVerlet(dt=dt)
    if mode == "overdamped":
        return mb.OverdampedLangevin(dt=dt, temperature=TEMPERATURE[wl], friction=FRICTION[wl])
    return mb.VelocityVerlet(dt=dt, coupling=andersen)


def run(wl, mode, steps, warmup):
    import torch
    import mollyb200 as mb
    dtype = np.float32
    sd, inters, _, dt, rc, label = bench.workload(wl, dtype)
    atoms = mb.atoms_from_arrays(sd["mass"], sd["charge"], sd["sigma"], sd["eps"], dtype)
    nf = mb.GPUNeighborFinder(dist_cutoff=bench.default_r_list(wl, rc), excluded_pairs=sd.get("excluded", np.zeros((0, 2), np.int32)) + 1,
                              special_pairs=sd.get("special", np.zeros((0, 2), np.int32)) + 1)
    specific = H.sixmrr_specific_lists(sd["golden"]) if "golden" in sd else ()
    s = mb.System(atoms=atoms, coords=torch.from_numpy(sd["coords"]).cuda().contiguous(), boundary=mb.CubicBoundary(*sd["box"]),
                  velocities=torch.from_numpy(sd["velocities"]).cuda().contiguous(), pairwise_inters=inters, neighbor_finder=nf,
                  dtype=dtype, specific_inter_lists=specific)
    sim = simulator(mode, dt, wl)
    rng = np.random.default_rng(1)
    mb.simulate(s, sim, warmup, rng=rng)
    rebuilds = s.stats()["n_rebuilds"]
    t0 = time.perf_counter()
    mb.simulate(s, sim, steps, init_step=warmup, rng=rng)  # the call ends in a device synchronise
    rate = steps / (time.perf_counter() - t0)
    st = s.stats()
    s.set_profiling(True)  # integration kernels only: their stage timer over a separate window
    mb.simulate(s, sim, PROF_STEPS, init_step=warmup + steps, rng=rng)
    integ_us = 1e3 * s.stats()["vv_ms"] / PROF_STEPS
    s.set_profiling(False)
    s.close()
    return rate, integ_us, label, (st["graph_mode"], st["n_rebuilds"] - rebuilds)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--warmup", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--workloads", default="c2,c3")
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()
    print(f"card: {card[0] if card else 'unknown'}")
    for wl in args.workloads.split(","):
        rates = {m: [] for m in MODES}
        integ = {m: [] for m in MODES}
        graphs = {}
        for _ in range(args.rounds):
            for m in MODES:
                r, us, label, graphs[m] = run(wl, m, args.steps, args.warmup)
                rates[m].append(r)
                integ[m].append(us)
        print(f"{wl}: {label}, {args.steps} timed steps, {args.rounds} alternating rounds")
        base = np.median(rates["vv"])
        for m in MODES:
            med = np.median(rates[m])
            print(f"  {m:15s} steps/s median {med:9.1f}  range {min(rates[m]):9.1f} - {max(rates[m]):9.1f}  "
                  f"({100.0 * (med / base - 1.0):+.1f} % vs vv)  graph_mode, rebuilds {graphs[m]}  "
                  f"integration kernels {np.median(integ[m]):6.1f} us/step")


if __name__ == "__main__":
    main()
