#!/usr/bin/env python
"""Temperature replica exchange on one GPU: aggregate replica-steps/s with the states' calls in one mb_simulate_group call
("group") against the same calls made one after another in the same process ("sequential"), for R replicas of

  readme: the reference's 100-atom LJ system (README.md:72-95), all-pairs;
  gb:     the 1170-atom GBN2 protein of tests/golden/6mrr_gb.npz, all-pairs, device state;
  c3:     6mrr in water (15 954 atoms) on the cell-list path.

Langevin (friction 1/ps, dt 2 fs), f32, temperatures spaced evenly from 300 K to 300 + 10 (R - 1) K. The modes alternate
over several rounds after a warm-up run (graph capture, first list build) and the median is reported. Also reported: the
host time per cycle spent outside the group call (energy evaluations for the exchange test, the decisions, velocity
scaling, parameter set-up), and the acceptance rate. The card's name and power limit are read in the same run.

    python scripts/bench_remd.py [--rounds 3] [--replicas 1,2,4,8,16] [--workloads readme,gb,c3]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "tests"), os.path.join(ROOT, "scripts"), ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)

# workload -> (steps per cycle, cycles per timed run)
PLAN = {"readme": (500, 4), "gb": (200, 4), "c3": (100, 3)}
DT = 0.002


def base_system(name):
    import mbhelpers as H
    import mollyb200 as mb
    if name == "readme":
        sd = H.readme_system(100, 2.0, seed=1)
        return H.make_system(sd, (mb.LennardJones(),), np.float32)
    if name == "gb":
        import bench_implicit_solvent as BI
        g = dict(np.load(os.path.join(ROOT, "tests", "golden", "6mrr_gb.npz")))
        return BI.system(g, True, False)
    g = dict(np.load(os.path.join(ROOT, "tests", "golden", "6mrr.npz")))
    return H.sixmrr_system(g, np.float32, r_list=1.2)


class Timed:
    """The engine runner, timing the calls that advance the replicas; sequential: one call at a time."""

    def __init__(self, sequential):
        from molly_jl_b200.api import _EngineRunner
        self.inner, self.sequential, self.t_run = _EngineRunner(), sequential, 0.0

    def run(self, repsys, calls, max_retries):
        t0 = time.perf_counter()
        if self.sequential:
            for s, call in calls:
                st = repsys.state_system(s)
                call.configure(st)
                call.run(st, max_retries)
        else:
            self.inner.run(repsys, calls, max_retries)
        self.t_run += time.perf_counter() - t0

    def energy(self, repsys, s, coords):
        return self.inner.energy(repsys, s, coords)


def replica_system(base, R):
    import mollyb200 as mb
    states = [mb.ThermoState(base, mb.Langevin(dt=DT, temperature=300.0 + 10.0 * k, friction=1.0)) for k in range(R)]
    x0 = base.coords
    copy = (lambda a: a.clone()) if hasattr(x0, "data_ptr") else (lambda a: a.copy())
    return mb.ReplicaSystem(states, [copy(x0) for _ in range(R)], replica_velocities=[copy(base.velocities) for _ in range(R)])


def measure(name, R, rounds):
    import mollyb200 as mb
    base = base_system(name)
    cyc, n_cyc = PLAN[name]
    sim = mb.ReplicaExchangeMD(DT, cyc * DT * 0.999999)  # (cycles of exactly cyc steps: n_cycles is a floor)
    rs = {mode: replica_system(base, R) for mode in ("group", "sequential")}
    rng = np.random.default_rng(7)
    for mode, r in rs.items():  # warm-up: graph capture and the first list build of every state's context
        mb.simulate_remd(r, sim, 2 * cyc, rng=rng, runner=Timed(mode == "sequential"))
    out = {m: [] for m in rs}
    host = []
    for _ in range(rounds):
        for mode, r in rs.items():
            t = Timed(mode == "sequential")
            t0 = time.perf_counter()
            mb.simulate_remd(r, sim, cyc * n_cyc, rng=rng, runner=t)
            wall = time.perf_counter() - t0
            out[mode].append(R * cyc * n_cyc / wall)
            if mode == "group":
                host.append(1e3 * (wall - t.t_run) / n_cyc)
    xl = rs["group"].exchange_logger
    acc = xl.n_exchanges / xl.n_attempts if xl.n_attempts else float("nan")
    for r in rs.values():
        r.close()
    base.close()
    g, s = statistics.median(out["group"]), statistics.median(out["sequential"])
    return dict(workload=name, R=R, group_replica_steps_per_s=round(g, 1), sequential_replica_steps_per_s=round(s, 1),
                speedup=round(g / s, 2), host_ms_per_cycle=round(statistics.median(host), 3), acceptance=round(acc, 3))


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unavailable ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--replicas", default="1,2,4,8,16")
    ap.add_argument("--workloads", default="readme,gb,c3")
    args = ap.parse_args()
    import mollyb200 as mb
    if mb.device_count() < 1:
        raise SystemExit("bench_remd needs a CUDA device: mollyb200 has no CPU fallback")
    print(json.dumps(dict(gpu=gpu_info())), flush=True)
    for name in args.workloads.split(","):
        for R in (int(r) for r in args.replicas.split(",")):
            print(json.dumps(measure(name, R, args.rounds)), flush=True)


if __name__ == "__main__":
    main()
