#!/usr/bin/env python
"""Cost of dissipative particle dynamics on the device: a Groot-Warren fluid (rho = 3, r_c = 1, a = 25, gamma = 4.5,
sigma = 3 so that kT = 1, lambda = 0.65, dt = 0.04, r_list = 1.5 r_c, unit masses, f32, device state) at N = 24 000 and
N = 192 000 on the cell-list path.

Two modes: "dpd" is DPDVelocityVerlet with the full DPDInteraction; "conservative" is the same term at gamma = sigma = 0,
for which the pair kernels neither gather v_j nor draw xi (other integrators refuse a DPD context). Both start from the
state the full DPD run reaches after the warm-up (random positions relax and the fluid reaches kT = 1), so both rebuild
the cell list about equally often, and the difference in steps/s and in the pair kernel's time per launch is the cost of
the gather, the draw and the dissipative and random arithmetic. The modes
alternate over several rounds and the median is reported. Prints steps/s of the timed window (captured step graphs) and,
from a second, profiled window of 200 steps (stream path, CUDA events around each launch), the pair kernel's time per
launch, with the card name and power limit read in the same run.

    python scripts/bench_dpd.py [--steps 2000] [--rounds 3] [--sizes 24000,192000]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

MODES = ("dpd", "conservative")
PROF_STEPS = 200
DT, LAM = 0.04, 0.65


def system(n, mode, x, v):
    import mollyb200 as mb
    g, s = (4.5, 3.0) if mode == "dpd" else (0.0, 0.0)
    inter = mb.DPDInteraction(a=25.0, gamma=g, sigma=s, r_c=1.0, dt=DT, use_neighbors=True, key=12345)
    atoms = mb.atoms_from_arrays(np.ones(n), np.zeros(n), np.zeros(n), np.zeros(n), np.float32)
    return mb.System(atoms, x, mb.CubicBoundary((n / 3.0) ** (1.0 / 3.0)), velocities=v, pairwise_inters=(inter,),
                     neighbor_finder=mb.GPUNeighborFinder(dist_cutoff=1.5), dtype=np.float32, k=1.0)


def equilibrated(n, warmup, seed=1):
    """Random positions and unit-variance velocities (device tensors) after `warmup` steps of the full DPD run."""
    import torch
    import mollyb200 as mb
    box = (n / 3.0) ** (1.0 / 3.0)
    r = np.random.default_rng(seed)
    x = torch.from_numpy(r.uniform(0, box, (n, 3)).astype(np.float32)).cuda()
    v = torch.from_numpy(r.normal(0, 1, (n, 3)).astype(np.float32)).cuda()
    s = system(n, "dpd", x, v)
    mb.simulate(s, mb.DPDVelocityVerlet(dt=DT, lam=LAM), warmup)
    s.close()
    return x, v


def run(n, mode, steps, start):
    import mollyb200 as mb
    s = system(n, mode, start[0].clone(), start[1].clone())
    sim = mb.DPDVelocityVerlet(dt=DT, lam=LAM)
    warmup = 50  # (graph capture and the first cell-list build)
    mb.simulate(s, sim, warmup)
    t0 = time.perf_counter()
    mb.simulate(s, sim, steps, init_step=warmup)  # the call ends in a device synchronise
    rate = steps / (time.perf_counter() - t0)
    st = s.stats()
    s.set_profiling(True)
    mb.simulate(s, sim, PROF_STEPS, init_step=warmup + steps)
    p = s.stats()
    pair_us = 1e3 * p["force_ms"] / (p["n_force_evals"] - st["n_force_evals"])
    s.set_profiling(False)
    s.close()
    return rate, pair_us, st["graph_mode"], st["path"], st["n_rebuilds"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--warmup", type=int, default=1000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--sizes", default="24000,192000")
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()
    print(f"card: {card[0] if card else 'unknown'}")
    for n in (int(v) for v in args.sizes.split(",")):
        rates = {m: [] for m in MODES}
        pair = {m: [] for m in MODES}
        info = {}
        start = equilibrated(n, args.warmup)
        for _ in range(args.rounds):
            for m in MODES:
                r, us, gm, path, nrb = run(n, m, args.steps, start)
                rates[m].append(r)
                pair[m].append(us)
                info[m] = (gm, path, nrb)
        print(f"N = {n}: {args.steps} timed steps after {args.warmup} steps of DPD, {args.rounds} alternating rounds")
        base = np.median(rates["conservative"])
        for m in MODES:
            med = np.median(rates[m])
            print(f"  {m:13s} steps/s median {med:9.1f}  range {min(rates[m]):9.1f} - {max(rates[m]):9.1f}  "
                  f"({100.0 * (med / base - 1.0):+.1f} % vs conservative)  pair kernel {np.median(pair[m]):7.1f} us/launch  "
                  f"graph_mode, path, rebuilds {info[m]}")


if __name__ == "__main__":
    main()
