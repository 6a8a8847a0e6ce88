#!/usr/bin/env python
"""Iterations per second of steepest-descent minimisation on the C3 and C2 workloads of bench.py (f32).

Two ways to run the same algorithm (simulators.jl:183-274), alternated over several rounds:
  device   mb_minimize_sd: every iteration on the device, one graph launch per call (tol 0: a fixed iteration count)
  python   the loop in Python over forces_energy calls (one evaluation per iteration, host coordinates): what a caller
           without the minimiser entry point does
Prints iterations/s for each, with the card name and power limit read in the same run.

    python scripts/bench_minimize.py [--iters 200] [--py-iters 40] [--rounds 3] [--workloads c3,c2]
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


def make_system(wl):
    import mollyb200 as mb
    dtype = np.float32
    sd, inters, _, _, rc, label = bench.workload(wl, dtype)
    atoms = mb.atoms_from_arrays(sd["mass"], sd["charge"], sd["sigma"], sd["eps"], dtype)
    nf = mb.GPUNeighborFinder(dist_cutoff=bench.default_r_list(wl, rc), excluded_pairs=sd.get("excluded", np.zeros((0, 2), np.int32)) + 1,
                              special_pairs=sd.get("special", np.zeros((0, 2), np.int32)) + 1)
    specific = H.sixmrr_specific_lists(sd["golden"]) if "golden" in sd else ()
    s = mb.System(atoms=atoms, coords=sd["coords"].copy(), boundary=mb.CubicBoundary(*sd["box"]), pairwise_inters=inters,
                  neighbor_finder=nf, dtype=dtype, specific_inter_lists=specific)
    return s, sd["box"], label


def python_loop(s, box, n, h=0.01):
    """The same loop over forces_energy: F, E of the trial together, kept forces on reject."""
    import mollyb200 as mb
    s.coords[...] = s.coords - np.floor(s.coords / box) * box
    F, E = mb.forces_energy(s)
    for _ in range(n):
        F64 = F.astype(np.float64)
        m = np.sqrt(np.max(np.einsum("ij,ij->i", F64, F64)))
        keep = s.coords.copy()
        x = s.coords.astype(np.float64) + h * F64 / m
        s.coords[...] = x - np.floor(x / box) * box
        F_t, E_t = mb.forces_energy(s)
        if E_t < E:
            h, E, F = 6 * h / 5, E_t, F_t
        else:
            s.coords[...] = keep
            h = h / 5
    return n


def run(wl, mode, iters, py_iters, warmup):
    import mollyb200 as mb
    s, box, label = make_system(wl)
    if mode == "device":
        mb.steepest_descent(s, mb.SteepestDescentMinimizer(max_steps=warmup, tol=0.0))  # capture, first build
        t0 = time.perf_counter()
        _, trace = mb.steepest_descent(s, mb.SteepestDescentMinimizer(max_steps=iters, tol=0.0))  # ends in a synchronise
        dt = time.perf_counter() - t0
        done, mode_used = len(trace) - 1, s.stats()["graph_mode"]
    else:
        python_loop(s, box, warmup)
        t0 = time.perf_counter()
        done = python_loop(s, box, py_iters)  # every forces_energy call ends in a synchronise
        dt = time.perf_counter() - t0
        mode_used = None
    s.close()
    return done / dt, label, mode_used


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--py-iters", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--workloads", default="c3,c2")
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()
    print(f"card: {card[0] if card else 'unknown'}")
    modes = ("device", "python")
    for wl in args.workloads.split(","):
        rates = {m: [] for m in modes}
        graph = None
        for _ in range(args.rounds):
            for m in modes:
                r, label, g = run(wl, m, args.iters, args.py_iters, args.warmup)
                rates[m].append(r)
                graph = g if g is not None else graph
        print(f"{wl}: {label}; device {args.iters} iterations per call (graph_mode {graph}), python {args.py_iters}; "
              f"{args.rounds} alternating rounds")
        for m in modes:
            print(f"  {m:7s} iterations/s median {np.median(rates[m]):9.1f}  range {min(rates[m]):9.1f} - {max(rates[m]):9.1f}")
        print(f"  device / python: {np.median(rates['device']) / np.median(rates['python']):.1f}x")


if __name__ == "__main__":
    main()
