"""Parent vs change, same inputs: checks that two builds of libmollyb200 compute the same thing.

    python scripts/compare_libs.py OLD.so NEW.so [--out DIR]

1. A fixed sequence of calls (forces, potential_energy, simulate with and without loggers; all-pairs, cell-list and 6mrr
   with bonded terms; graph and stream step paths) runs once with each library in a fresh process; kernel_launches,
   n_force_evals and graph_mode from stats() after every call must be identical.
2. bench.py --workload c2 / c3 --dump-outputs with each library: C2 coordinates and velocities must be bit-identical. C3 adds
   bonded forces with float atomics, so the OLD library runs it twice and the OLD-vs-NEW difference must lie within
   twice that run-to-run difference.
Libraries are given relative to molly.jl_b200/ or as paths. Needs a CUDA device."""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _stats_sequence():
    sys.path[:0] = [os.path.join(ROOT, "tests"), ROOT]
    import mbhelpers as H
    import mollyb200 as mb
    g = dict(np.load(os.path.join(ROOT, "tests", "golden", "6mrr.npz")))
    lj = lambda nl: (mb.LennardJones(cutoff=mb.ShiftedForceCutoff(1.0), use_neighbors=nl),)
    systems = {
        "allpairs-f64": lambda: H.make_system(H.lj_fluid(6, dtype=np.float64), lj(False), np.float64),
        "brick-f32": lambda: H.make_system(H.lj_fluid(8, dtype=np.float32), lj(True), np.float32, r_list=1.2),
        "6mrr-f64": lambda: H.sixmrr_system(g, np.float64, r_list=1.2, dispersion=True),
    }
    rec = {}
    for name, make in systems.items():
        s = make()
        dt = 0.0005 if name.startswith("6mrr") else 0.002
        seq = []

        def snap(label):
            st = s.stats()
            seq.append([label, st["kernel_launches"], st["n_force_evals"], st["graph_mode"]])

        mb.forces(s), snap("forces")
        mb.potential_energy(s), snap("potential_energy")
        mb.simulate(s, mb.VelocityVerlet(dt=dt), 20), snap("simulate graph")
        s.loggers = {"pe": mb.PotentialEnergyLogger(5), "x": mb.CoordinatesLogger(7), "v": mb.VelocitiesLogger(3)}
        mb.simulate(s, mb.VelocityVerlet(dt=dt), 20), snap("simulate graph + loggers")
        mb.simulate(s, mb.VelocityVerlet(dt=dt, remove_CM_motion=2), 20), snap("simulate stream + loggers")
        s.loggers = {}
        mb.simulate(s, mb.VelocityVerlet(dt=dt, remove_CM_motion=2), 10), snap("simulate stream")
        rec[name] = seq
        s.close()
    print(json.dumps(rec))


def _lib(p):
    return p if os.path.isabs(p) else os.path.join(ROOT, "molly.jl_b200", p)


def _run(env_lib, args):
    env = dict(os.environ, MOLLYB200_LIB=env_lib)
    r = subprocess.run([sys.executable] + args, cwd=ROOT, env=env, capture_output=True, text=True)
    if r.returncode != 0:
        raise SystemExit(f"{args} with {env_lib} failed:\n{r.stderr[-3000:]}")
    return r.stdout


def main():
    old, new = _lib(sys.argv[1]), _lib(sys.argv[2])
    out = sys.argv[sys.argv.index("--out") + 1] if "--out" in sys.argv else os.path.join("/tmp", "compare_libs")
    ok = True
    stats = {lib: json.loads(_run(lib, [__file__, "--stats-child"]).strip().splitlines()[-1]) for lib in (old, new)}
    for name in stats[old]:
        same = stats[old][name] == stats[new][name]
        ok &= same
        print(f"[stats {name}] {'identical' if same else 'DIFFERENT'}: {stats[old][name]}" +
              ("" if same else f" vs {stats[new][name]}"))
    bench = ["bench.py", "--no-cpu-baseline", "--no-e2e", "--steps", "200", "--warmup", "20"]
    dumps = {}
    for wl, runs in (("c2", [("old", old), ("new", new)]), ("c3", [("old", old), ("old2", old), ("new", new)])):
        for tag, lib in runs:
            d = os.path.join(out, f"{wl}-{tag}")
            _run(lib, bench + ["--workload", wl, "--dump-outputs", d])
            dumps[wl, tag] = {k: np.load(os.path.join(d, f"{k}.npy")) for k in ("coords", "velocities")}
    for k in ("coords", "velocities"):
        same = np.array_equal(dumps["c2", "old"][k], dumps["c2", "new"][k])
        ok &= same
        print(f"[c2 {k}] {'bit-identical' if same else 'DIFFERENT'}")
        spread = np.abs(dumps["c3", "old"][k] - dumps["c3", "old2"][k]).max()
        diff = np.abs(dumps["c3", "old"][k] - dumps["c3", "new"][k]).max()
        within = diff <= 2 * spread
        ok &= within
        print(f"[c3 {k}] max|old-new|={diff:.3e}, run-to-run max|old-old|={spread:.3e}: {'within' if within else 'OUTSIDE'}")
    print("compare_libs:", "OK" if ok else "MISMATCH")
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    if "--stats-child" in sys.argv:
        _stats_sequence()
    else:
        main()
