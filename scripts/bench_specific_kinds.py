#!/usr/bin/env python
"""Cost of position restraints on the C3 workload of bench.py (6mrr, LJ + CRF + bonds/angles/torsions, VelocityVerlet +
Andersen, f32, device state), next to the same run without them.

"c3" is the workload as bench.py runs it; "c3+restraints" adds a HarmonicPositionRestraint (k = 1000 kJ mol^-1 nm^-2) on
every protein heavy atom through add_position_restraints, the usual restrained equilibration. The protein is the atoms up
to the last one in a torsion (the waters have none), heavy means a mass above 1.5 g/mol. The two runs alternate over
several rounds and the median of the rounds is reported, with the card name and power limit read in the same run. Then the
mean device time per launch of bonded_kernel from a separate torch.profiler run of 200 steps.

    python scripts/bench_specific_kinds.py [--steps 1000] [--rounds 3] [--no-profile]
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

MODES = ("c3", "c3+restraints")
K_RESTRAINT = 1000.0


def make_system(mode):
    import torch
    import mollyb200 as mb
    dtype = np.float32
    sd, inters, _, dt, rc, label = bench.workload("c3", dtype)
    g = sd["golden"]
    atoms = mb.atoms_from_arrays(sd["mass"], sd["charge"], sd["sigma"], sd["eps"], dtype)
    nf = mb.GPUNeighborFinder(dist_cutoff=bench.default_r_list("c3", rc), excluded_pairs=sd["excluded"] + 1,
                              special_pairs=sd["special"] + 1)
    s = mb.System(atoms=atoms, coords=torch.from_numpy(sd["coords"]).cuda().contiguous(), boundary=mb.CubicBoundary(*sd["box"]),
                  velocities=torch.from_numpy(sd["velocities"]).cuda().contiguous(), pairwise_inters=inters, neighbor_finder=nf,
                  dtype=dtype, specific_inter_lists=H.sixmrr_specific_lists(g))
    n_res = 0
    if mode == "c3+restraints":
        n_protein = int(max(g["proper_idx"].max(), g["improper_idx"].max())) + 1
        heavy = np.flatnonzero(np.asarray(sd["mass"])[:n_protein] > 1.5) + 1
        s = mb.add_position_restraints(s, K_RESTRAINT, atom_selector=heavy, restrain_coords=sd["coords"])
        n_res = len(heavy)
    return s, mb.VelocityVerlet(dt=dt, coupling=mb.AndersenThermostat(300.0, 1.0)), label, n_res


def run(mode, steps, warmup):
    import mollyb200 as mb
    s, sim, label, n_res = make_system(mode)
    rng = np.random.default_rng(1)
    mb.simulate(s, sim, warmup, rng=rng)
    t0 = time.perf_counter()
    mb.simulate(s, sim, steps, init_step=warmup, rng=rng)  # the call ends in a device synchronise
    rate = steps / (time.perf_counter() - t0)
    graph = s.stats()["graph_mode"]
    s.close()
    return rate, label, n_res, graph


def profile(mode, steps=200):
    """Mean device time per launch (us) and launches per step of bonded_kernel."""
    import torch
    from torch.profiler import ProfilerActivity, profile as tprofile
    import mollyb200 as mb
    s, sim, _, _ = make_system(mode)
    mb.simulate(s, sim, 50, rng=np.random.default_rng(1))
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        mb.simulate(s, sim, steps, init_step=50, rng=np.random.default_rng(1))
        torch.cuda.synchronize()
    s.close()
    t, c = 0.0, 0
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and "bonded_kernel<" in e.name:
            t, c = t + e.device_time, c + 1
    return (t / c if c else float("nan")), c / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--warmup", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--no-profile", action="store_true")
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()
    print(f"card: {card[0] if card else 'unknown'}")
    rates = {m: [] for m in MODES}
    info = {}
    for _ in range(args.rounds):
        for m in MODES:
            r, label, n_res, graph = run(m, args.steps, args.warmup)
            rates[m].append(r)
            info[m] = (n_res, graph)
    print(f"{label}, {args.steps} timed steps, {args.rounds} alternating rounds")
    base = np.median(rates["c3"])
    for m in MODES:
        med = np.median(rates[m])
        print(f"  {m:14s} steps/s median {med:9.1f}  range {min(rates[m]):9.1f} - {max(rates[m]):9.1f}  "
              f"({100.0 * (med / base - 1.0):+.1f} % vs c3)  restrained atoms {info[m][0]}  graph_mode {info[m][1]}")
    if not args.no_profile:
        for m in MODES:
            us, per_step = profile(m)
            print(f"  {m:14s} bonded_kernel {us:.2f} us per launch, {per_step:.2f} launches per step")


if __name__ == "__main__":
    main()
