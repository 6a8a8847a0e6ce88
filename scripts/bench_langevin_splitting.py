#!/usr/bin/env python
"""Cost of LangevinSplitting next to VelocityVerlet and Langevin, on the C2 and C3 workloads of bench.py (f32, device state).

The same number of steps with VelocityVerlet, Langevin (friction 1 ps^-1), LangevinSplitting "BAOAB" and "OBABO" and the
deterministic "BAB", alternated over several rounds; the median of the rounds is reported. The splitting's friction is a
mass per time: FRICTION gives 1 ps^-1 for argon (C2) and for carbon (C3). The baths target the temperature the workload
starts at, so that the neighbour-list rebuild rate stays that of the uncoupled run. Prints steps/s and the rebuilds of the
timed window for each, with the card name and power limit read in the same run, then the mean device time per launch of
each integration kernel from a separate torch.profiler run of 200 steps.

    python scripts/bench_langevin_splitting.py [--steps 1000] [--rounds 3] [--workloads c2,c3] [--no-profile]
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

MODES = ("vv", "langevin", "BAOAB", "OBABO", "BAB")
TEMPERATURE = {"c2": 90.0, "c3": 300.0}  # K: what tests/mbhelpers.lj_fluid and the 6mrr velocities are drawn at
FRICTION = {"c2": 39.948, "c3": 12.011}  # g mol^-1 ps^-1: 1 ps^-1 for argon and for carbon
KERNELS = ("vv_kick_drift_kernel", "vv_kick2_kernel", "langevin_step_kernel", "split_pass_kernel", "brick_force_kernel")


def simulator(mode, dt, wl):
    import mollyb200 as mb
    if mode == "vv":
        return mb.VelocityVerlet(dt=dt)
    if mode == "langevin":
        return mb.Langevin(dt=dt, temperature=TEMPERATURE[wl], friction=1.0)
    return mb.LangevinSplitting(dt=dt, temperature=TEMPERATURE[wl], friction=FRICTION[wl], splitting=mode)


def make_system(wl):
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
    return s, dt, label


def run(wl, mode, steps, warmup):
    import mollyb200 as mb
    s, dt, label = make_system(wl)
    sim = simulator(mode, dt, wl)
    rng = np.random.default_rng(1)
    mb.simulate(s, sim, warmup, rng=rng)
    rebuilds = s.stats()["n_rebuilds"]
    t0 = time.perf_counter()
    mb.simulate(s, sim, steps, init_step=warmup, rng=rng)  # the call ends in a device synchronise
    rate = steps / (time.perf_counter() - t0)
    st = s.stats()
    s.close()
    return rate, label, (st["graph_mode"], st["n_rebuilds"] - rebuilds)


def profile(wl, mode, steps=200):
    """Mean device time per launch (us) and launches per step of each integration kernel and the pair kernel."""
    import torch
    from torch.profiler import ProfilerActivity, profile as tprofile
    import mollyb200 as mb
    s, dt, _ = make_system(wl)
    sim = simulator(mode, dt, wl)
    mb.simulate(s, sim, 50, rng=np.random.default_rng(1))
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        mb.simulate(s, sim, steps, init_step=50, rng=np.random.default_rng(1))
        torch.cuda.synchronize()
    s.close()
    out = {}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        for k in KERNELS:
            if k + "<" in e.name:
                t, c = out.get(k, (0.0, 0))
                out[k] = (t + e.device_time, c + 1)
    return {k: (t / c, c / steps) for k, (t, c) in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--warmup", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--workloads", default="c2,c3")
    ap.add_argument("--no-profile", action="store_true")
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()
    print(f"card: {card[0] if card else 'unknown'}")
    for wl in args.workloads.split(","):
        rates = {m: [] for m in MODES}
        graphs = {}
        for _ in range(args.rounds):
            for m in MODES:
                r, label, graphs[m] = run(wl, m, args.steps, args.warmup)
                rates[m].append(r)
        print(f"{wl}: {label}, {args.steps} timed steps, {args.rounds} alternating rounds")
        base = np.median(rates["vv"])
        for m in MODES:
            med = np.median(rates[m])
            print(f"  {m:9s} steps/s median {med:9.1f}  range {min(rates[m]):9.1f} - {max(rates[m]):9.1f}  "
                  f"({100.0 * (med / base - 1.0):+.1f} % vs vv)  graph_mode, rebuilds {graphs[m]}")
        if args.no_profile:
            continue
        for m in MODES:
            k = profile(wl, m)
            print(f"  {wl} {m:9s} kernels (us per launch, launches per step): " +
                  ", ".join(f"{name} {t:.2f} x {c:.2f}" for name, (t, c) in sorted(k.items())))


if __name__ == "__main__":
    main()
