#!/usr/bin/env python
"""Cost of the generalized-Born implicit solvent (ImplicitSolventGBN2) in f32 Langevin dynamics (friction 1 ps^-1,
device state), on 6mrr without water (1170 atoms, tests/golden/6mrr_gb.npz) and on eight copies of it 10 nm apart
(9360 atoms), both in a 100 nm box with LJ + Coulomb at 5 nm and the bonded terms, as the reference's implicit-solvent
system is built. The 1170-atom system is run twice: with the pairs on the cell-list path (neighbour list at 5.5 nm) and on
the all-pairs path. The eight copies run on the all-pairs path only: at a 5.5 nm list radius the cell-list path's halo of
the eight copies does not fit in shared memory. The GB kernels are the same on both paths; only the atom order differs
(spatially sorted slots on the cell-list path, input order on the all-pairs path).

For each system: steps/s with and without the GB term (median of alternating rounds), the GB kernels' device time per
step from a separate torch.profiler run, and GB pair evaluations per second (3 passes x N^2 ordered pairs per step over
that kernel time). The card name, power limit and max SM clock are read in the same run.

    python scripts/bench_implicit_solvent.py [--steps 2000] [--rounds 3] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "tests"), ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)


def replicate(g, copies):
    """The fixture's system `copies` times (2 x 2 x 2 for 8), each copy shifted by 10 nm per grid step."""
    n = len(g["coords"])
    shifts = [np.array([i, j, k]) * 10.0 for i in range(2) for j in range(2) for k in range(2)][:copies]
    out = {}
    out["coords"] = np.concatenate([g["coords"] + s for s in shifts])
    for k in ("mass", "charge", "sigma", "eps", "gbn2_offset_radii", "gbn2_scaled_offset_radii", "gbn2_alpha", "gbn2_beta",
              "gbn2_gamma", "gbn2_neck_class"):
        out[k] = np.concatenate([g[k]] * copies)
    for k in ("excluded", "special", "bond_idx", "angle_idx", "proper_idx", "improper_idx"):
        out[k] = np.concatenate([g[k] + c * n for c in range(copies)])
    for k in ("bond_par", "angle_par", "proper_par", "improper_par"):
        out[k] = np.concatenate([g[k]] * copies)
    for k in ("box", "lj14scale", "coulomb14scale", "gbn2_d0", "gbn2_m0", "gbn2_offset", "kappa"):
        out[k] = g[k]
    return out


def system(g, with_gb, cell_list, dtype=np.float32):
    import torch

    import mbhelpers as H
    import mollyb200 as mb
    n = len(g["coords"])
    gb = mb.ImplicitSolventGBN2(offset_radii=g["gbn2_offset_radii"], scaled_offset_radii=g["gbn2_scaled_offset_radii"],
                                alpha=g["gbn2_alpha"], beta=g["gbn2_beta"], gamma=g["gbn2_gamma"], neck_class=g["gbn2_neck_class"],
                                d0=g["gbn2_d0"], m0=g["gbn2_m0"], offset=float(g["gbn2_offset"]), kappa=float(g["kappa"]))
    atoms = mb.atoms_from_arrays(g["mass"], g["charge"], g["sigma"], g["eps"], dtype)
    inters = (mb.LennardJones(cutoff=mb.DistanceCutoff(5.0), use_neighbors=cell_list, weight_special=float(g["lj14scale"])),
              mb.Coulomb(cutoff=mb.DistanceCutoff(5.0), use_neighbors=cell_list, weight_special=float(g["coulomb14scale"])))
    nf = mb.GPUNeighborFinder(dist_cutoff=5.5 if cell_list else 0.0, excluded_pairs=g["excluded"] + 1,
                              special_pairs=g["special"] + 1)
    v = np.random.default_rng(1).normal(0, 0.3, (n, 3))
    x = torch.tensor(g["coords"], dtype=torch.float32, device="cuda")
    vt = torch.tensor(v, dtype=torch.float32, device="cuda")
    return mb.System(atoms=atoms, coords=x, boundary=mb.CubicBoundary(*g["box"]), velocities=vt, pairwise_inters=inters,
                     neighbor_finder=nf, dtype=dtype, specific_inter_lists=H.sixmrr_specific_lists(g),
                     general_inters=(gb,) if with_gb else ())


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unavailable ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch

    import mollyb200 as mb
    g0 = dict(np.load(os.path.join(ROOT, "tests", "golden", "6mrr_gb.npz")))
    sim = mb.Langevin(dt=0.002, temperature=300.0, friction=1.0)
    results = {"gpu": gpu_info()}
    print("gpu:", results["gpu"])
    g8 = replicate(g0, 8)
    for label, g, cell_list in (("6mrr_nowater x1, cell-list pairs", g0, True), ("6mrr_nowater x1, all-pairs pairs", g0, False),
                                ("6mrr_nowater x8, all-pairs pairs", g8, False)):
        n = len(g["coords"])
        systems = {k: system(g, k, cell_list) for k in (False, True)}
        for s in systems.values():
            mb.simulate(s, sim, 200, rng=np.random.default_rng(0))  # warm-up: build, capture the graph
        rates = {False: [], True: []}
        for _ in range(a.rounds):
            for k, s in systems.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                mb.simulate(s, sim, a.steps, rng=np.random.default_rng(0))
                torch.cuda.synchronize()
                rates[k].append(a.steps / (time.perf_counter() - t0))
        med = {k: float(np.median(v)) for k, v in rates.items()}
        # GB kernel time per step: a separate profiled run
        s = systems[True]
        prof_steps = 200
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            mb.simulate(s, sim, prof_steps, rng=np.random.default_rng(0))
            torch.cuda.synchronize()
        gb = {e.key: e.device_time_total / prof_steps for e in prof.key_averages() if "gb_" in e.key}
        gb_us = sum(gb.values())
        pair_evals = 3.0 * n * (n - 1)
        r = dict(n_atoms=n, steps_per_s_with_gb=med[True], steps_per_s_without_gb=med[False],
                 rounds_with=rates[True], rounds_without=rates[False], gb_kernel_us_per_step=gb_us,
                 gb_us_per_kernel={k.split("(")[0]: v for k, v in gb.items()},
                 gb_pair_evals_per_s=pair_evals / (gb_us * 1e-6) if gb_us > 0 else None, path=s.stats()["path"],
                 graph_mode=s.stats()["graph_mode"])
        results[label] = r
        print(label, json.dumps(r))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_implicit_solvent.json"), "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
