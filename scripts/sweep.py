#!/usr/bin/env python
"""Tuning sweep on the GPU box: force-kernel / rebuild stage times for several brick shapes.
    python scripts/sweep.py --workload c2 --configs 0,0,0 3,3,3 4,4,4 ...   (bx,by,bz; 0,0,0 = auto)"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "tests"), ROOT):
    sys.path.insert(0, p)
import bench  # noqa: E402
import mbhelpers as H  # noqa: E402
import mollyb200 as mb  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="c2")
    ap.add_argument("--configs", nargs="+", default=["0,0,0"])
    ap.add_argument("--r-list", type=float, nargs="+", default=[None])
    ap.add_argument("--steps", type=int, default=100)
    args = ap.parse_args()
    sd, inters, ointers, dt, rc, label = bench.workload(args.workload, np.float32)
    atoms = mb.atoms_from_arrays(sd["mass"], sd["charge"], sd["sigma"], sd["eps"], np.float32)
    for rl in args.r_list:
        r_list = rl if rl is not None else rc + 0.1
        for cfg in args.configs:
            bx, by, bz = [int(v) for v in cfg.split(",")]
            nf = mb.GPUNeighborFinder(dist_cutoff=r_list, excluded_pairs=sd.get("excluded", np.zeros((0, 2), np.int32)) + 1,
                                      special_pairs=sd.get("special", np.zeros((0, 2), np.int32)) + 1, n_steps=0)
            specific = H.sixmrr_specific_lists(sd["golden"]) if "golden" in sd else ()
            s = mb.System(atoms=atoms, coords=sd["coords"].copy(), boundary=mb.CubicBoundary(*sd["box"]),
                          velocities=sd["velocities"].copy(), pairwise_inters=inters, neighbor_finder=nf, dtype=np.float32,
                          specific_inter_lists=specific)
            s.engine()
            try:
                s.set_launch_config((bx, by, bz))
                sim = mb.VelocityVerlet(dt=dt)
                mb.simulate(s, sim, 20)
                t0 = time.perf_counter()
                mb.simulate(s, sim, args.steps, init_step=20)
                wall = time.perf_counter() - t0
                st_g = s.stats()
                s.set_profiling(True)
                mb.simulate(s, sim, args.steps, init_step=20 + args.steps)
                st = s.stats()
                s.set_profiling(False)
                out = dict(cfg=cfg, r_list=r_list, brick=st["brick_dims"], bricks=st["n_bricks"], halo=st["max_halo"],
                           stride=st["list_stride"], maxnb=st["max_neighbors"], graph_mode=st_g["graph_mode"],
                           wall_us_per_step=1e6 * wall / args.steps,
                           force_us=1e3 * st["force_ms"] / max(st["force_launches"], 1),
                           vv_us=1e3 * st["vv_ms"] / max(st["vv_launches"], 1),
                           rebuild_ms_total=st["rebuild_ms"], rebuilds=st["n_rebuilds"] - st_g["n_rebuilds"])
                print(json.dumps(out), flush=True)
            except Exception as e:  # keep sweeping
                print(json.dumps(dict(cfg=cfg, r_list=r_list, error=str(e))), flush=True)
            s.close()


if __name__ == "__main__":
    main()
