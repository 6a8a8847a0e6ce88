"""Parent vs change, same inputs: checks that two builds of libmollyb200 compute the same thing.

    python scripts/compare_libs.py OLD.so NEW.so [--out DIR]

1. A fixed sequence of calls (forces, potential_energy, simulate with and without loggers; all-pairs, cell-list and 6mrr
   with bonded terms; graph and stream step paths) runs once with each library in a fresh process; kernel_launches,
   n_force_evals and graph_mode from stats() after every call must be identical.
2. Integration and minimisation runs, each on a fresh context, in a fresh process per library: VelocityVerlet (plain,
   Immediate, Berendsen, Bussi with n_steps 1 and 5, Andersen), Langevin, NoseHoover, MTSIntegrator with 2 and 3 levels,
   MTSLangevinIntegrator and LangevinSplitting (BAOAB, OBABO, ABOBA, BAB) under remove_CM_motion 0, 1, 3 and init_step 0,
   7, each integrator with all six device loggers, a SteepestDescentMinimizer run and random_velocities; on all-pairs and
   brick systems, f32 and f64, graph and stream (MOLLYB200_NO_GRAPH=1) paths. The systems have no bonded terms, so the
   inner MTS levels carry zero forces and no float atomics enter: coordinates, velocities, logger histories and the
   minimiser trace must be bit-identical, and the stats after every run identical.
3. bench.py --workload c2 / c3 --dump-outputs with each library: C2 coordinates and velocities must be bit-identical. C3 adds
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


def _run_sequence(out):
    """Every run of item 2 on a fresh context; its outputs go to the npz `out`, its stats to stdout as JSON."""
    sys.path[:0] = [os.path.join(ROOT, "tests"), ROOT]
    import mbhelpers as H
    import mollyb200 as mb
    lj = lambda nl: (mb.LennardJones(cutoff=mb.ShiftedForceCutoff(1.0), use_neighbors=nl),)
    systems = {"allpairs": (6, False, 0.0), "brick": (8, True, 1.2)}
    dt = 0.002

    def mts(cls, fractions, *args):
        def make(cm):
            sim = cls(dt, *args, pi_fractions=(1,), remove_CM_motion=cm)
            sim.ordered_fractions = fractions  # levels that hold no term: (1,) alone would run as VelocityVerlet
            return sim
        return make

    integrators = {
        "vv": lambda cm: mb.VelocityVerlet(dt=dt, remove_CM_motion=cm),
        "langevin": lambda cm: mb.Langevin(dt=dt, temperature=100.0, friction=2.0, remove_CM_motion=cm),
        "nosehoover": lambda cm: mb.NoseHoover(dt=dt, temperature=100.0, remove_CM_motion=cm),
        "mts2": mts(mb.MTSIntegrator, (1, 2)),
        "mts3": mts(mb.MTSIntegrator, (1, 2, 4)),
        "mtslangevin": mts(mb.MTSLangevinIntegrator, (1, 2), 100.0, 2.0),
    }
    for splitting in ("BAOAB", "OBABO", "ABOBA", "BAB"):
        integrators[f"split-{splitting}"] = lambda cm, sp=splitting: mb.LangevinSplitting(dt, 100.0, 80.0, sp, remove_CM_motion=cm)
    couplings = {"immediate": mb.ImmediateThermostat(120.0), "berendsen": mb.BerendsenThermostat(120.0, 0.05),
                 "bussi1": mb.VelocityRescaleThermostat(120.0, 0.05), "bussi5": mb.VelocityRescaleThermostat(120.0, 0.05, 5),
                 "andersen": mb.AndersenThermostat(120.0, 0.05)}
    arrays, stats = {}, {}
    for (sname, (cells, nl, r_list)) in systems.items():
        for dtype in (np.float32, np.float64):
            for path in ("graph", "stream"):
                if path == "stream":
                    os.environ["MOLLYB200_NO_GRAPH"] = "1"
                else:
                    os.environ.pop("MOLLYB200_NO_GRAPH", None)
                base = f"{sname}-{np.dtype(dtype).name}-{path}"

                def run(label, fn, loggers=None):
                    s = H.make_system(H.lj_fluid(cells, dtype=dtype), lj(nl), dtype, r_list=r_list)
                    s.loggers = loggers or {}
                    extra = fn(s)
                    key = f"{base}:{label}"
                    arrays[key + ":coords"] = np.array(s.coords)
                    arrays[key + ":velocities"] = np.array(s.velocities)
                    for name, lg in s.loggers.items():
                        arrays[key + f":log-{name}"] = np.asarray(mb.values(lg), np.float64)
                    if extra is not None:
                        arrays[key + ":extra"] = np.asarray(extra)
                    st = s.stats()
                    stats[key] = [st["kernel_launches"], st["n_force_evals"], st["graph_mode"]]
                    s.close()

                def sim(s, integ, init=0):
                    mb.simulate(s, integ, 20, init_step=init, rng=np.random.default_rng(1))

                for iname, make in integrators.items():
                    for cm in (0, 1, 3):
                        for init in (0, 7):
                            run(f"{iname}-cm{cm}-init{init}", lambda s: sim(s, make(cm), init))
                    loggers = lambda: {"pe": mb.PotentialEnergyLogger(5), "ke": mb.KineticEnergyLogger(3),
                                       "te": mb.TotalEnergyLogger(4), "T": mb.TemperatureLogger(2),
                                       "x": mb.CoordinatesLogger(7), "v": mb.VelocitiesLogger(3)}
                    run(f"{iname}-loggers", lambda s: sim(s, make(1)), loggers())
                for cname, c in couplings.items():
                    run(f"vv-{cname}", lambda s: sim(s, mb.VelocityVerlet(dt=dt, coupling=c)))
                run("minimize", lambda s: mb.steepest_descent(s, mb.SteepestDescentMinimizer(0.01, 40, 1.0))[1])
                run("random_velocities", lambda s: mb.random_velocities(s, 100.0, rng=np.random.default_rng(3)))
    os.environ.pop("MOLLYB200_NO_GRAPH", None)
    np.savez(out, **arrays)
    print(json.dumps(stats))


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
    os.makedirs(out, exist_ok=True)
    runs = {}
    for tag, lib in (("old", old), ("new", new)):
        npz = os.path.join(out, f"runs-{tag}.npz")
        runs[tag] = (json.loads(_run(lib, [__file__, "--runs-child", npz]).strip().splitlines()[-1]), np.load(npz))
    (st_old, a_old), (st_new, a_new) = runs["old"], runs["new"]
    n_diff = 0
    for key in sorted(set(a_old.files) | set(a_new.files)):
        same = key in a_old.files and key in a_new.files and np.array_equal(a_old[key], a_new[key], equal_nan=True)
        if not same:
            n_diff += 1
            print(f"[runs {key}] DIFFERENT")
    for key in sorted(set(st_old) | set(st_new)):
        if st_old.get(key) != st_new.get(key):
            n_diff += 1
            print(f"[runs {key}] stats DIFFERENT: {st_old.get(key)} vs {st_new.get(key)}")
    ok &= n_diff == 0
    print(f"[runs] {len(st_old)} runs, {len(a_old.files)} arrays: " + ("bit-identical, identical stats" if n_diff == 0 else f"{n_diff} differences"))
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
    elif "--runs-child" in sys.argv:
        _run_sequence(sys.argv[sys.argv.index("--runs-child") + 1])
    else:
        main()
