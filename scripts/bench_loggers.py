#!/usr/bin/env python
"""Cost of logging energies during a VelocityVerlet run, on the C2 and C3 workloads of bench.py (f32, device state).

Three ways to run the same number of steps, alternated over several rounds:
  none     simulate(n) without loggers
  in-run   simulate(n) with TotalEnergyLogger(10) + TemperatureLogger(10), recorded on the device
  chunked  simulate(10) repeatedly, with potential_energy + kinetic_energy between the calls (the way without loggers)
Prints steps/s for each, with the card name and power limit read in the same run.

    python scripts/bench_loggers.py [--steps 1000] [--rounds 3] [--workloads c2,c3]
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


def make_system(wl, loggers):
    import torch
    import mollyb200 as mb
    dtype = np.float32
    sd, inters, _, dt, rc, label = bench.workload(wl, dtype)
    atoms = mb.atoms_from_arrays(sd["mass"], sd["charge"], sd["sigma"], sd["eps"], dtype)
    nf = mb.GPUNeighborFinder(dist_cutoff=bench.default_r_list(wl, rc), excluded_pairs=sd.get("excluded", np.zeros((0, 2), np.int32)) + 1,
                              special_pairs=sd.get("special", np.zeros((0, 2), np.int32)) + 1)
    xs = torch.from_numpy(sd["coords"]).cuda().contiguous()
    vs = torch.from_numpy(sd["velocities"]).cuda().contiguous()
    specific = H.sixmrr_specific_lists(sd["golden"]) if "golden" in sd else ()
    s = mb.System(atoms=atoms, coords=xs, boundary=mb.CubicBoundary(*sd["box"]), velocities=vs, pairwise_inters=inters,
                  neighbor_finder=nf, dtype=dtype, specific_inter_lists=specific, loggers=loggers)
    coupling = mb.AndersenThermostat(300.0, 1.0) if wl == "c3" else None
    return s, mb.VelocityVerlet(dt=dt, coupling=coupling), label


def run(wl, mode, steps, warmup):
    import mollyb200 as mb
    loggers = {"e": mb.TotalEnergyLogger(10), "t": mb.TemperatureLogger(10)} if mode == "in-run" else None
    s, sim, label = make_system(wl, loggers)
    rng = np.random.default_rng(1)

    def go(n, init):
        if mode == "chunked":
            for k in range(0, n, 10):
                mb.simulate(s, sim, 10, init_step=init + k, rng=rng)
                mb.potential_energy(s)
                mb.kinetic_energy(s)
        else:
            mb.simulate(s, sim, n, init_step=init, rng=rng)

    go(warmup, 0)
    t0 = time.perf_counter()
    go(steps, warmup)  # every call ends in a device synchronise
    dt = time.perf_counter() - t0
    extra = len(s.loggers["e"].history) if loggers else 0
    s.close()
    return steps / dt, label, extra


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
    modes = ("none", "in-run", "chunked")
    for wl in args.workloads.split(","):
        rates = {m: [] for m in modes}
        for _ in range(args.rounds):
            for m in modes:
                r, label, _ = run(wl, m, args.steps, args.warmup)
                rates[m].append(r)
        print(f"{wl}: {label}, {args.steps} timed steps, {args.rounds} alternating rounds")
        base = np.median(rates["none"])
        for m in modes:
            med = np.median(rates[m])
            print(f"  {m:8s} steps/s median {med:9.1f}  range {min(rates[m]):9.1f} - {max(rates[m]):9.1f}  "
                  f"({100.0 * (med / base - 1.0):+.1f} % vs none)")


if __name__ == "__main__":
    main()
