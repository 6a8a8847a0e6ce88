"""GPU tests of the multiple-time-step integrators (src/simulators.jl:1616-1940): f64 trajectory parity of MTSIntegrator and
MTSLangevinIntegrator with the numpy restatement of mts_substeps! (tests/mts_oracle.py) on 6mrr with bonded terms (cell-list
path, with a rebuild inside the run), a triclinic all-pairs box with bonded terms, 6mrr + PME on the stream path and a level
whose list is empty; remove_CM_motion x init_step and chunked calls; the pair kernel once per outer step (host counter and
profiler); the observer / determinism properties of the step graph; the O step's moments; and a temperature protocol
adapted from the reference's test/simulation.jl MTSLangevinIntegrator test."""
import ctypes as C
import math

import numpy as np
import pytest

import mbhelpers as H
import mollyb200 as mb
import mts_oracle as mo
import thermostat_oracle as tho
from oracle import bonded as bd
from oracle import oracle as o
from test_gpu_parity import _pos_err

pytestmark = pytest.mark.gpu

F32, F64 = np.float32, np.float64
KB = mb.BOLTZMANN_K
_FN = {2: bd.bond_forces, 3: bd.angle_forces, 4: bd.torsion_forces}


def _keys(seed):
    r = np.random.default_rng(seed)
    return tho.rng_words(int(r.integers(0, 2 ** 63)), int(r.integers(0, 2 ** 63)))


def _level_forces(sim, pair_fe, lists, box):
    """Per-level forces of the reference's mts_interaction_groups: level 0 = pairs (+ PME inside pair_fe) and the lists at
    fraction 1; level l = the lists at ordered_fractions[l]. lists: (idx 0-based, par) in si_fractions order."""
    def make(level):
        mine = [(idx, par) for (idx, par), f in zip(lists, sim.si_fractions) if sim.ordered_fractions.index(f) == level]

        def fe(x):
            f = pair_fe(x) if level == 0 else np.zeros_like(x)
            for idx, par in mine:
                if len(idx):
                    f = f + _FN[idx.shape[1]](x, box, idx, par)[0]
            return f
        return fe
    return [make(level) for level in range(len(sim.ordered_fractions))]


def _sixmrr_lists(g):
    return [(g["bond_idx"], g["bond_par"]), (g["angle_idx"], g["angle_par"]),
            (np.concatenate([g["proper_idx"], g["improper_idx"]]), np.concatenate([g["proper_par"], g["improper_par"]]))]


def _sim(kind, dt, si, pi=(1, 1), gi=(), rcm=1, T=300.0, friction=10.0):
    if kind == "mts":
        return mb.MTSIntegrator(dt, pi_fractions=pi, si_fractions=si, gi_fractions=gi, remove_CM_motion=rcm)
    return mb.MTSLangevinIntegrator(dt, T, friction, pi_fractions=pi, si_fractions=si, gi_fractions=gi, remove_CM_motion=rcm)


def _parity(s, sd, sim, levels, n, seed=7, init_step=0, wrap=None, label="", tol=(1e-9, 1e-8)):
    lang = (KB * sim.temperature, sim.friction, _keys(seed)) if isinstance(sim, mb.MTSLangevinIntegrator) else None
    box = sd["box"]
    x_ref, v_ref = mo.simulate_mts(levels, sd["coords"], sd["velocities"], sd["mass"], sim.dt, n, sim.ordered_fractions,
                                   wrap or (lambda x: x - np.floor(x / box) * box), remove_cm_every=sim.remove_CM_motion,
                                   init_step=init_step, langevin=lang)
    rb0 = s.stats()["n_rebuilds"] if s._ctx is not None else 0
    mb.simulate(s, sim, n, init_step=init_step, rng=np.random.default_rng(seed))
    st = s.stats()
    ex, ev = _pos_err(s.coords, x_ref, box), np.abs(s.velocities - v_ref).max()
    print(f"[{type(sim).__name__} {sim.ordered_fractions} {label} rcm={sim.remove_CM_motion} init={init_step} path={st['path']} "
          f"graph={st['graph_mode']} rebuilds={st['n_rebuilds'] - rb0}] dx={ex:.3e} dv={ev:.3e}")
    assert ex < tol[0] and ev < tol[1]
    return st, st["n_rebuilds"] - rb0


KINDS = ["mts", "mts-langevin"]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("si", [(2, 2, 1), (4, 2, 1), (8, 4, 2)])
def test_parity_6mrr_bonded_celllist(golden_6mrr, kind, si):
    """6mrr (15 954 atoms) with bonds, angles and torsions at their own levels, 20 outer steps of 2 fs. A 0.05 nm skin makes
    the neighbour structure rebuild inside the run."""
    g = golden_6mrr
    s = H.sixmrr_system(g, F64, r_list=1.05)
    orc, sd = H.sixmrr_oracle(g)
    sim = _sim(kind, 0.002, si)
    levels = _level_forces(sim, lambda x: orc.forces_nl(x, orc.neighbor_list(x, 1.05), energy=False)[0], _sixmrr_lists(g), sd["box"])
    st, rebuilds = _parity(s, sd, sim, levels, 20, label="6mrr")
    assert st["path"] == 1 and rebuilds >= 1
    s.close()


def _molecules(n_mol=100, L=2.4, triclinic=False, dtype=F64):
    """H.molecular_system with bonds, angles and a torsion per molecule (test_gpu_triclinic_bonded's lists), LJ + CRF with
    exclusions and 1-4 specials, all-pairs path. triclinic: the sheared box (L,0,0), (L,L,0), (-L,0,L), the same lattice
    as the cube of side L, so the rectangular oracle gives its forces."""
    from test_gpu_triclinic_bonded import _chain_lists
    sd = H.molecular_system(n_mol, [L, L, L], seed=3, stable=True)
    sd["box"] = np.asarray(sd["box"], np.float64)
    lists = _chain_lists(n_mol)
    inters = (mb.LennardJones(cutoff=mb.DistanceCutoff(1.0), use_neighbors=True, weight_special=0.5),
              mb.CoulombReactionField(dist_cutoff=1.0, use_neighbors=True, weight_special=0.8333))
    atoms = mb.atoms_from_arrays(sd["mass"], sd["charge"], sd["sigma"], sd["eps"], dtype)
    nf = mb.GPUNeighborFinder(dist_cutoff=1.2, excluded_pairs=sd["excluded"] + 1, special_pairs=sd["special"] + 1)
    bnd = mb.TriclinicBoundary([L, 0, 0], [L, L, 0], [-L, 0, L]) if triclinic else mb.CubicBoundary(L, L, L)
    s = mb.System(atoms=atoms, coords=sd["coords"].astype(dtype), velocities=sd["velocities"].astype(dtype), boundary=bnd,
                  pairwise_inters=inters, neighbor_finder=nf, dtype=dtype, specific_inter_lists=lists)
    orc = H.make_oracle(sd, [o.Inter(o.LJ, o.CUT_DISTANCE, 1.0, weight_special=0.5, use_neighbors=True),
                             o.Inter(o.CRF, o.CUT_DISTANCE, 1.0, weight_special=0.8333, use_neighbors=True)])
    ol = [(np.stack([li.is_, li.js] + ([li.ks] if hasattr(li, "ks") else []) + ([li.ls] if hasattr(li, "ls") else []), 1).astype(int) - 1,
           li.arrays()[1]) for li in lists]
    return sd, s, (lambda x: orc.forces_allpairs(x, energy=False)[0]), ol


@pytest.mark.parametrize("kind", KINDS)
def test_parity_triclinic_allpairs_bonded(kind):
    sd, s, pair_fe, lists = _molecules(triclinic=True)
    sim = _sim(kind, 0.002, (4, 2, 1), T=120.0)
    st, _ = _parity(s, sd, sim, _level_forces(sim, pair_fe, lists, sd["box"]), 30, label="triclinic")
    assert st["path"] == 0
    s.close()


@pytest.mark.parametrize("kind", KINDS)
def test_parity_6mrr_pme_stream_path(golden_6mrr, kind):
    from oracle import pme
    g = golden_6mrr
    s = H.sixmrr_pme_system(g, F64)
    sd = H.sixmrr_description(g)
    alpha = pme.pme_alpha(1.0)
    orc = H.make_oracle(sd, [o.Inter(o.LJ, o.CUT_DISTANCE, 1.0, weight_special=float(g["lj14scale"]), use_neighbors=True),
                             o.Inter(o.EWALD_REAL, o.CUT_DISTANCE, 1.0, weight_special=float(g["coulomb14scale"]), ewald_alpha=alpha,
                                     use_neighbors=True)])
    excl = np.concatenate([g["excluded"], g["special"]])

    def pair_fe(x):
        f = orc.forces_nl(x, orc.neighbor_list(x, 1.2), energy=False)[0]
        return f + pme.pme_reciprocal(x, g["charge"], sd["box"], r_cut=1.0, error_tol=0.0005, order=5)[0] + \
            pme.ewald_exclusion(x, g["charge"], sd["box"], excl)[0]
    sim = _sim(kind, 0.002, (2, 2, 1), gi=(1, 4))  # (LJDispersionCorrection exerts no force: any fraction)
    st, _ = _parity(s, sd, sim, _level_forces(sim, pair_fe, _sixmrr_lists(g), sd["box"]), 10, label="6mrr+PME")
    assert st["graph_mode"] == 0
    s.close()


@pytest.mark.parametrize("kind", KINDS)
def test_parity_level_with_empty_list(golden_6mrr, kind):
    """An empty bond list at the innermost level (fraction 4): the innermost substeps drift with zero forces."""
    g = golden_6mrr
    lists = H.sixmrr_specific_lists(g) + (mb.InteractionList2Atoms([], [], [], []),)
    sd0 = H.sixmrr_description(g)
    atoms = mb.atoms_from_arrays(sd0["mass"], sd0["charge"], sd0["sigma"], sd0["eps"], F64)
    ref = H.sixmrr_system(g, F64)
    s = mb.System(atoms=atoms, coords=ref.coords, velocities=ref.velocities, boundary=ref.boundary, pairwise_inters=ref.pairwise_inters,
                  neighbor_finder=ref.neighbor_finder, dtype=F64, specific_inter_lists=lists)
    orc, sd = H.sixmrr_oracle(g)
    sim = _sim(kind, 0.002, (2, 2, 1, 4))
    ol = _sixmrr_lists(g) + [(np.zeros((0, 2), int), np.zeros((0, 2)))]
    _parity(s, sd, sim, _level_forces(sim, lambda x: orc.forces_nl(x, orc.neighbor_list(x, 1.2), energy=False)[0], ol, sd["box"]),
            10, label="empty level")
    s.close()


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("rcm,init_step", [(0, 0), (1, 0), (3, 0), (0, 13), (1, 13), (3, 13)])
def test_parity_remove_cm_and_init_step(kind, rcm, init_step):
    sd, s, pair_fe, lists = _molecules()
    sim = _sim(kind, 0.002, (4, 2, 1), rcm=rcm, T=120.0)
    _parity(s, sd, sim, _level_forces(sim, pair_fe, lists, sd["box"]), 20, init_step=init_step, label="molecules")
    s.close()


@pytest.mark.parametrize("kind", KINDS)
def test_chunked_calls_equal_one_call(kind):
    """simulate(10) then simulate(10; init_step=10) == simulate(20): the reference recomputes F_0 at the start of a call,
    which equals the forces the long call carries over; the draws depend on (keys, outer step, substep, atom) only."""
    sim = _sim(kind, 0.002, (4, 2, 1), T=120.0)
    sd, a, _, _ = _molecules()
    _, b, _, _ = _molecules()
    mb.simulate(a, sim, 20, rng=np.random.default_rng(1))
    mb.simulate(b, sim, 10, rng=np.random.default_rng(1))
    mb.simulate(b, sim, 10, init_step=10, rng=np.random.default_rng(1))
    assert _pos_err(a.coords, b.coords, sd["box"]) < 1e-12 and np.abs(a.velocities - b.velocities).max() < 1e-12
    a.close(); b.close()


def _lj_brick(dtype=F64):
    sd = H.lj_fluid(6, seed=3, dtype=dtype)
    return sd, H.make_system(sd, (mb.LennardJones(cutoff=mb.ShiftedForceCutoff(0.9), use_neighbors=True),), dtype, r_list=0.92)


def test_one_level_is_velocity_verlet_bit_identical():
    sd, a = _lj_brick()
    _, b = _lj_brick()
    mb.simulate(a, mb.MTSIntegrator(0.002, pi_fractions=(1,)), 40)
    mb.simulate(b, mb.VelocityVerlet(0.002), 40)
    assert np.array_equal(a.coords, b.coords) and np.array_equal(a.velocities, b.velocities)
    assert a.stats()["graph_mode"] == 1
    a.close(); b.close()


def test_one_level_6mrr_equals_velocity_verlet(golden_6mrr):
    g = golden_6mrr
    a, b = H.sixmrr_system(g, F64), H.sixmrr_system(g, F64)
    mb.simulate(a, mb.MTSIntegrator(0.002, pi_fractions=(1, 1), si_fractions=(1, 1, 1)), 20)
    mb.simulate(b, mb.VelocityVerlet(0.002), 20)
    assert _pos_err(a.coords, b.coords, g["box"]) < 1e-12 and np.abs(a.velocities - b.velocities).max() < 1e-11
    a.close(); b.close()


@pytest.mark.parametrize("no_graph", ["0", "1"])
def test_pair_kernel_once_per_outer_step(golden_6mrr, monkeypatch, no_graph):
    """Unlogged: n_force_evals grows by n_steps + 1, and the profiler sees n_steps + 1 pair-kernel launches and as many
    bonded_kernel launches as the reference evaluates each level: fractions (1, 2) with torsions at level 0 and bonds and
    angles at level 1 give n + 1 level-0 launches and 3 n level-1 launches."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    monkeypatch.setenv("MOLLYB200_NO_GRAPH", no_graph)
    g = golden_6mrr
    s = H.sixmrr_system(g, F32)
    sim = mb.MTSIntegrator(0.002, pi_fractions=(1, 1), si_fractions=(2, 2, 1))
    mb.simulate(s, sim, 4)  # (first build and graph capture outside the window)
    n = 12
    ev0 = s.stats()["n_force_evals"]
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        mb.simulate(s, sim, n)
        torch.cuda.synchronize()
    st = s.stats()
    names = [e.name for e in prof.events()]
    pair = sum(1 for x in names if "brick_force_kernel<" in x)
    bonded = sum(1 for x in names if "bonded_kernel<" in x)
    print(f"[MTS launches graph={st['graph_mode']}] force evals +{st['n_force_evals'] - ev0}, pair kernels {pair}, bonded {bonded}")
    assert st["graph_mode"] == (0 if no_graph == "1" else 1)
    assert st["n_force_evals"] - ev0 == n + 1
    assert pair == n + 1 and bonded == (n + 1) + 3 * n
    s.close()


def _run(kind="mts", seed=2, n=30, loggers=None, device=False, si=(4, 2, 1)):
    sd, s, _, _ = _molecules()
    if loggers:
        s.loggers = loggers
    if device:
        import torch
        s.coords, s.velocities = torch.from_numpy(s.coords).cuda(), torch.from_numpy(s.velocities).cuda()
    mb.simulate(s, _sim(kind, 0.002, si, T=120.0), n, rng=np.random.default_rng(seed))
    out = [a.cpu().numpy() if hasattr(a, "cpu") else a.copy() for a in (s.coords, s.velocities)] + [s.stats()["graph_mode"]]
    s.close()
    return out


def _close(a, b, box=2.4):
    return _pos_err(a[0], b[0], np.full(3, box)) < 1e-12 and np.abs(a[1] - b[1]).max() < 1e-12


@pytest.mark.parametrize("kind", KINDS)
def test_logged_equals_unlogged(kind):
    a = _run(kind)
    lg = {"v": mb.VelocitiesLogger(7), "e": mb.TotalEnergyLogger(5), "x": mb.CoordinatesLogger(10)}
    b = _run(kind, loggers=lg)
    assert _close(a, b)
    assert len(lg["e"].history) == len(mb.record_steps(5, 30)) and len(lg["v"].history) == len(mb.record_steps(7, 30))
    c = _run(kind, n=21)
    assert np.abs(lg["v"].history[3] - c[1]).max() < 1e-12  # the record at step 21 = a run stopped there


@pytest.mark.parametrize("kind", KINDS)
def test_graph_equals_stream_path(kind, monkeypatch):
    res = []
    for no_graph in ("0", "1"):
        monkeypatch.setenv("MOLLYB200_NO_GRAPH", no_graph)
        res.append(_run(kind))
    assert (res[0][2], res[1][2]) == (1, 0)
    assert _close(res[0], res[1])


@pytest.mark.parametrize("kind", KINDS)
def test_host_equals_device_buffers(kind):
    assert _close(_run(kind), _run(kind, device=True))


def test_velocity_verlet_after_mts_equals_fresh_system(golden_6mrr):
    g = golden_6mrr
    s = H.sixmrr_system(g, F64)
    mb.simulate(s, mb.MTSIntegrator(0.002, pi_fractions=(1, 1), si_fractions=(4, 2, 1)), 10)
    ref = H.sixmrr_system(g, F64, coords=s.coords.copy(), velocities=s.velocities.copy())
    mb.simulate(s, mb.VelocityVerlet(0.001), 20, init_step=10)
    mb.simulate(ref, mb.VelocityVerlet(0.001), 20, init_step=10)
    assert _pos_err(s.coords, ref.coords, g["box"]) < 1e-12 and np.abs(s.velocities - ref.velocities).max() < 1e-10
    s.close(); ref.close()


@pytest.mark.parametrize("dtype", [F32, F64])
def test_o_step_statistics_free_particles(dtype):
    """No forces (eps = 0, an empty bond list at fraction 4): every innermost substep is v <- c v + sigma xi with
    c = exp(-dt friction / 4). After k outer steps, E[v] = c^(4k) v0 and Var[v] = (kT/m)(1 - c^(8k)). The bars are 5 standard
    errors of the sample mean and variance; massless atoms keep c^(4k) v0."""
    n_grp, masses = 6000, [1.0, 12.0, 39.948, 200.0]
    n = n_grp * len(masses) + 50
    mass = np.concatenate([np.full(n_grp, m) for m in masses] + [np.zeros(50)])
    rng = np.random.default_rng(4)
    x = rng.random((n, 3)) * 10.0
    v0 = np.tile(np.array([0.7, -0.3, 0.2]), (n, 1))
    T, gamma, dt = 300.0, 5.0, 0.004
    kT, c = KB * T, math.exp(-gamma * dt / 4)
    atoms = mb.atoms_from_arrays(mass, np.zeros(n), np.full(n, 0.3), np.zeros(n), dtype)
    s = mb.System(atoms=atoms, coords=x.astype(dtype), velocities=v0.astype(dtype), boundary=mb.CubicBoundary(10.0),
                  pairwise_inters=(mb.LennardJones(),), dtype=dtype, specific_inter_lists=(mb.InteractionList2Atoms([], [], [], []),))
    sim = mb.MTSLangevinIntegrator(dt, T, gamma, pi_fractions=(1,), si_fractions=(4,), remove_CM_motion=0)
    done = 0
    for k in (1, 10, 60):
        mb.simulate(s, sim, k - done, init_step=done, rng=np.random.default_rng(11))
        done = k
        v = s.velocities.astype(np.float64)
        for gi, m in enumerate(masses):
            vg = v[gi * n_grp:(gi + 1) * n_grp] - c ** (4 * k) * v0[0]
            var = kT / m * (1 - c ** (8 * k))
            N = vg.size
            assert abs(vg.mean()) < 5 * math.sqrt(var / N), (k, m)
            assert abs(vg.var() / var - 1) < 5 * math.sqrt(2 / N), (k, m)
        np.testing.assert_allclose(v[-50:], np.tile(c ** (4 * k) * v0[0], (50, 1)), rtol=1e-5 if dtype == F32 else 1e-12)
    s.close()


@pytest.mark.parametrize("dtype", [F32, F64])
def test_temperature_protocol(golden_6mrr, dtype):
    """Adapted from test/simulation.jl:1306-1395 (MTSLangevinIntegrator on TIP4P water with virtual sites and a CRescale
    barostat, neither of which the engine has): 6mrr, 1 fs outer step, friction 10 ps^-1, si_fractions (4, 4, 2),
    TemperatureLogger(10), 1000 outer steps; the mean temperature after the first 80 records lies in [290, 310] K."""
    g = golden_6mrr
    s = H.sixmrr_system(g, dtype)
    s.loggers = {"temperature": mb.TemperatureLogger(10)}
    mb.simulate(s, mb.MTSLangevinIntegrator(0.001, 300.0, 10.0, pi_fractions=(1, 1), si_fractions=(4, 4, 2)), 1000,
                rng=np.random.default_rng(5))
    temps = np.array(mb.values(s.loggers["temperature"]))
    assert len(temps) == 101
    print(f"[MTSLangevin protocol {np.dtype(dtype).name}] <T> after 80 records = {temps[80:].mean():.2f} K")
    assert 290.0 < temps[80:].mean() < 310.0
    s.close()


def test_refusals_leave_coordinates_untouched():
    sd, s, _, _ = _molecules()
    ctx = s.engine()
    L = s._L
    x, v = s.coords.copy(), s.velocities.copy()

    def params(**kw):
        p = mb.capi.MBMTSParams()
        p.dt, p.n_steps, p.remove_cm_every, p.n_levels = 0.002, 10, 1, 2
        p.fractions[:2] = (1, 2)
        for k, val in kw.items():
            if k == "fractions":
                p.fractions[:len(val)] = val
            else:
                setattr(p, k, val)
        return p
    bad = [params(dt=0.0), params(n_steps=-1), params(n_levels=0), params(n_levels=9), params(fractions=(2, 4)),
           params(fractions=(1, 1)), params(fractions=(1, 3, 5), n_levels=3),
           params(langevin=1, kT=-1.0), params(langevin=1, kT=2.0, friction=math.nan), params(fractions=(1, 2048))]
    for p in bad:
        assert L.mb_simulate_mts(ctx, s.coords.ctypes.data, s.velocities.ctypes.data, C.byref(p), None) == mb.capi.MB_ERR_INVALID
        assert np.array_equal(x, s.coords) and np.array_equal(v, s.velocities)
    # a term at a level the call does not have
    lv = np.full(300, 2, np.int32)
    assert L.mb_set_specific_levels(ctx, 0, 300, lv.ctypes.data) == 0
    assert L.mb_simulate_mts(ctx, s.coords.ctypes.data, s.velocities.ctypes.data, C.byref(params()), None) == mb.capi.MB_ERR_INVALID
    assert L.mb_set_specific_levels(ctx, 0, 299, lv.ctypes.data) == mb.capi.MB_ERR_INVALID
    # a velocity coupling set on the context
    assert L.mb_set_velocity_coupling(ctx, C.byref(mb.capi.MBVCoupling(mb.capi.MB_VC_IMMEDIATE, 0, 2.0, 0.0))) == 0
    p = params(n_levels=3, fractions=(1, 2, 4))
    assert L.mb_simulate_mts(ctx, s.coords.ctypes.data, s.velocities.ctypes.data, C.byref(p), None) == mb.capi.MB_ERR_INVALID
    assert b"velocity coupling" in L.mb_last_error()
    assert np.array_equal(x, s.coords) and np.array_equal(v, s.velocities)
    mb.simulate(s, _sim("mts", 0.002, (4, 2, 1)), 5)  # simulate clears the coupling and sets the levels: the run goes through
    s.close()
