"""GPU tests of the generalized-Born implicit solvent (ImplicitSolventOBC / ImplicitSolventGBN2, mb_set_implicit_solvent):
the reference's "Implicit solvent" test (test/protein.jl:663-707) on 6mrr without water against OpenMM, including the GBN2
minimisation; GB-only parity with the numpy oracle (tests/gbsa_oracle.py) in f64 and f32 on the all-pairs path, the
cell-list path (with a rebuild that reorders the slots), a cutoff and a triclinic box; f64 trajectories of VelocityVerlet,
Langevin, NoseHoover and MTS against numpy loops over oracle forces; determinism, graph = stream, logged = unlogged and
re-setting the parameters; the engine's refusals."""
import ctypes as C
import os

import numpy as np
import pytest

import gbsa_oracle as gbo
import langevin_oracle as lo
import mbhelpers as H
import mollyb200 as mb
import mts_oracle as mo
import nosehoover_oracle as nho
import thermostat_oracle as tho

pytestmark = pytest.mark.gpu

F32, F64 = np.float32, np.float64
KB = mb.BOLTZMANN_K
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def g():
    return np.load(os.path.join(ROOT, "tests", "golden", "6mrr_gb.npz"))


def _inter(g, model, idx=None, **over):
    """The engine's GB interaction for `model` (optionally for the atoms idx only), and the oracle's."""
    p = gbo.from_golden(g, model, **over)
    sel = (lambda a: np.asarray(a)[idx]) if idx is not None else (lambda a: np.asarray(a))
    kw = dict(offset_radii=sel(p.offset_radii), scaled_offset_radii=sel(p.scaled_offset_radii), kappa=p.kappa,
              offset=p.offset, dist_cutoff=p.dist_cutoff, use_ACE=p.use_ace)
    if model == "gbn2":
        gb = mb.ImplicitSolventGBN2(alpha=sel(p.alpha), beta=sel(p.beta), gamma=sel(p.gamma), neck_class=sel(p.neck_class),
                                    d0=p.d0, m0=p.m0, **kw)
    else:
        gb = mb.ImplicitSolventOBC(alpha=1.0, beta=0.8, gamma=4.85, **kw)
    if idx is not None:
        for k in ("offset_radii", "scaled_offset_radii", "alpha", "beta", "gamma"):
            setattr(p, k, sel(getattr(p, k)))
        if p.has_neck:
            p.neck_class = sel(p.neck_class)
    return gb, p


def _full_system(g, model, dtype, coords=None, velocities=None, loggers=None):
    """System(6mrr_nowater.pdb, ff99SBildn; boundary 100 nm, dist_cutoff 5 nm, nonbonded_method :none, implicit_solvent,
    kappa 1 nm^-1) as test/protein.jl:668-679 builds it."""
    gb, _ = _inter(g, model)
    atoms = mb.atoms_from_arrays(g["mass"], g["charge"], g["sigma"], g["eps"], dtype)
    inters = (mb.LennardJones(cutoff=mb.DistanceCutoff(5.0), use_neighbors=True, weight_special=float(g["lj14scale"])),
              mb.Coulomb(cutoff=mb.DistanceCutoff(5.0), use_neighbors=True, weight_special=float(g["coulomb14scale"])))
    nf = mb.GPUNeighborFinder(dist_cutoff=5.5, excluded_pairs=g["excluded"] + 1, special_pairs=g["special"] + 1)
    x = g["coords"] if coords is None else coords
    v = np.zeros_like(g["coords"]) if velocities is None else velocities
    return mb.System(atoms=atoms, coords=np.asarray(x).astype(dtype), boundary=mb.CubicBoundary(*g["box"]),
                     velocities=np.asarray(v).astype(dtype), pairwise_inters=inters, neighbor_finder=nf, dtype=dtype,
                     specific_inter_lists=H.sixmrr_specific_lists(g), general_inters=(gb,), loggers=loggers)


def _full_oracle(g, model):
    from test_gbsa_oracle import pair_forces_energy
    _, p = _inter(g, model)

    def fe(x):
        return (gbo.forces_energy(x, g["charge"], p, box=g["box"])[0] + pair_forces_energy(g, x)[0]
                + H.bonded_forces_oracle(g, x)[0])
    return fe


@pytest.mark.parametrize("model", ["obc2", "gbn2"])
def test_reference_implicit_solvent(g, model):
    s = _full_system(g, model, F64)
    f = mb.forces(s)
    f2, e2 = mb.forces_energy(s)
    e = mb.potential_energy(s)
    df = np.linalg.norm(f - g[f"forces_{model}"], axis=1).max()
    de = abs(e - float(g[f"energy_{model}"]))
    print(f"[{model} f64 path={s.stats()['path']}] max |dF| = {df:.2e} kJ/mol/nm, |dE| = {de:.2e} kJ/mol")
    assert df < 1e-3 and de < 1e-2
    # (the bonded terms add with atomics, so the full system agrees to rounding, as forces vs forces_virial in the reference)
    assert np.abs(f - f2).max() < 1e-10 and abs(e - e2) < 1e-8
    if model == "gbn2":
        x0 = s.coords.copy()
        mb.simulate(s, mb.SteepestDescentMinimizer(tol=400.0))
        e_min = mb.potential_energy(s)
        rmsd = np.sqrt(np.mean(np.sum((s.coords - x0) ** 2, axis=1)))
        print(f"[gbn2 minimised] E {e:.3f} -> {e_min:.3f} kJ/mol, rmsd {rmsd:.4f} nm")
        assert e_min < e and rmsd < 0.1


def _gb_only(g, model, dtype, idx=None, box=None, tric=None, brick=False, coords=None, **over):
    """A system with the GB term alone: no pairwise interactions (all-pairs path), or a zero-epsilon LJ on a neighbour
    list (cell-list path; it adds no force)."""
    gb, p = _inter(g, model, idx, **over)
    sel = (lambda a: np.asarray(a)[idx]) if idx is not None else (lambda a: np.asarray(a))
    n = len(p.offset_radii)
    x = sel(g["coords"]) if coords is None else coords
    if tric is not None:
        boundary = mb.TriclinicBoundary(*tric.bv)
        x = np.array([tric.wrap(c) for c in x])
    else:
        boundary = mb.CubicBoundary(*box)
        x = x - np.floor(x / box) * box
    atoms = mb.atoms_from_arrays(sel(g["mass"]), sel(g["charge"]), np.full(n, 0.3), np.zeros(n), dtype)
    inters, nf = (), None
    if brick:
        inters = (mb.LennardJones(cutoff=mb.DistanceCutoff(1.0), use_neighbors=True),)
        nf = mb.GPUNeighborFinder(dist_cutoff=1.2, excluded_pairs=np.zeros((0, 2), np.int32), special_pairs=np.zeros((0, 2), np.int32))
    s = mb.System(atoms=atoms, coords=x.astype(dtype), boundary=boundary, pairwise_inters=inters, neighbor_finder=nf,
                  dtype=dtype, general_inters=(gb,))
    return s, p, x, sel(g["charge"])


def _check(s, p, x, q, dtype, label, box=None, tric=None, path=None):
    f_ref, e_ref = gbo.forces_energy(x, q, p, box=box, tric=tric)
    f, e = mb.forces_energy(s)
    fmax = np.abs(f_ref).max()
    err, eerr = np.abs(f - f_ref).max(), abs(e - e_ref)
    st = s.stats()
    print(f"[{label} {np.dtype(dtype).name} path={st['path']}] max|dF| = {err:.3e} (tol {H.tol(dtype, fmax):.1e}, max|F| {fmax:.1f}) "
          f"|dE| = {eerr:.3e} (tol {H.etol(dtype, e_ref):.1e}, E {e_ref:.3f})")
    if path is not None:
        assert st["path"] == path
    assert err <= H.tol(dtype, fmax) and eerr <= H.etol(dtype, e_ref)


CASES = ["allpairs", "kappa0", "no-ace", "cutoff", "triclinic", "brick"]


@pytest.mark.parametrize("dtype", [F64, F32])
@pytest.mark.parametrize("model", ["obc2", "gbn2"])
@pytest.mark.parametrize("case", CASES)
def test_gb_only_oracle_parity(g, model, dtype, case):
    from oracle.triclinic import Triclinic
    box = np.array([7.0, 7.0, 7.0])
    kw, tric, idx = {}, None, None
    if case == "kappa0":
        kw = dict(kappa=0.0)
    elif case == "no-ace":
        kw = dict(use_ace=False)
    elif case == "cutoff":
        kw = dict(dist_cutoff=1.2)
    elif case == "triclinic":
        tric = Triclinic(np.array([[3.0, 0, 0], [0.6, 3.1, 0], [0.4, -0.5, 3.2]]))
        idx = np.argsort(np.linalg.norm(g["coords"] - g["coords"][0], axis=1), kind="stable")[:400]
        kw = dict(dist_cutoff=1.2)
    s, p, x, q = _gb_only(g, model, dtype, idx=idx, box=None if tric else box, tric=tric, brick=case == "brick", **kw)
    _check(s, p, x, q, dtype, f"{model} {case}", box=None if tric else box, tric=tric, path=1 if case == "brick" else 0)
    if case == "brick":  # a move that forces a rebuild, which reorders the slots
        x2 = x + np.random.default_rng(3).normal(0, 0.3, x.shape)
        x2 = x2 - np.floor(x2 / box) * box
        s.coords = x2.astype(dtype)
        rb = s.stats()["n_rebuilds"]
        _check(s, p, x2, q, dtype, f"{model} brick after move", box=box, path=1)
        assert s.stats()["n_rebuilds"] > rb


def _keys(seed):
    r = np.random.default_rng(seed)
    return tho.rng_words(int(r.integers(0, 2 ** 63)), int(r.integers(0, 2 ** 63)))


@pytest.mark.parametrize("integ", ["vv", "langevin", "nosehoover", "mts"])
def test_dynamics_f64(g, integ):
    n, dt, T = 20, 0.001, 300.0
    v0 = np.random.default_rng(11).normal(0, 0.3, g["coords"].shape)
    s = _full_system(g, "gbn2", F64, velocities=v0)
    fe = _full_oracle(g, "gbn2")
    box = g["box"]
    wrap = lambda x: x - np.floor(x / box) * box  # noqa: E731
    x0 = wrap(g["coords"])
    if integ == "vv":
        x_ref, v_ref = mo.simulate_mts([fe], x0, v0, g["mass"], dt, n, (1,), wrap)
        mb.simulate(s, mb.VelocityVerlet(dt=dt), n)
    elif integ == "langevin":
        x_ref, v_ref = lo.simulate_langevin(fe, x0, v0, g["mass"], dt, n, KB * T, 1.0, _keys(5), wrap)
        mb.simulate(s, mb.Langevin(dt=dt, temperature=T, friction=1.0), n, rng=np.random.default_rng(5))
    elif integ == "nosehoover":
        x_ref, v_ref, _ = nho.simulate_nose_hoover(fe, x0, v0, g["mass"], dt, n, KB * T, 100 * dt, wrap)
        mb.simulate(s, mb.NoseHoover(dt=dt, temperature=T, damping=100 * dt), n)
    else:  # GB and the pairs at level 0, the bonded lists at fraction 2
        _, p = _inter(g, "gbn2")
        from test_gbsa_oracle import pair_forces_energy

        def f0(x):
            return gbo.forces_energy(x, g["charge"], p, box=box)[0] + pair_forces_energy(g, x)[0]

        def f1(x):
            return H.bonded_forces_oracle(g, x)[0]
        sim = mb.MTSIntegrator(dt, pi_fractions=(1, 1), si_fractions=(2, 2, 2), gi_fractions=(1,))
        x_ref, v_ref = mo.simulate_mts([f0, f1], x0, v0, g["mass"], dt, n, sim.ordered_fractions, wrap)
        mb.simulate(s, sim, n)
    st = s.stats()
    ex = np.abs(((s.coords - x_ref) + box / 2) % box - box / 2).max()
    ev = np.abs(s.velocities - v_ref).max()
    print(f"[{integ} gbn2 path={st['path']} graph={st['graph_mode']}] dx={ex:.3e} dv={ev:.3e}")
    assert st["graph_mode"] == 1
    assert ex < 1e-9 and ev < 1e-8


def _gb_dyn(g, dtype, loggers=None, brick=True, **over):
    """The GB term alone, by default on the cell-list path (a zero-epsilon LJ drives the list): no atomics anywhere in the
    step."""
    box = np.array([7.0, 7.0, 7.0])
    s, p, x, q = _gb_only(g, "gbn2", dtype, box=box, brick=brick, **over)
    s.velocities = np.random.default_rng(2).normal(0, 0.3, x.shape).astype(dtype)
    s.loggers = dict(loggers or {})
    return s


@pytest.mark.parametrize("dtype", [F64, F32])
def test_determinism_and_graph_rules(g, monkeypatch, dtype):
    s = _gb_dyn(g, dtype)
    a, b = mb.forces_energy(s), mb.forces_energy(s)
    assert np.array_equal(a[0], b[0]) and a[1] == b[1]
    out = {}
    for key, no_graph, logged in (("graph", "0", False), ("stream", "1", False), ("logged", "0", True)):
        monkeypatch.setenv("MOLLYB200_NO_GRAPH", no_graph)
        s = _gb_dyn(g, dtype, loggers={"pe": mb.PotentialEnergyLogger(5), "x": mb.CoordinatesLogger(5)} if logged else None)
        mb.simulate(s, mb.Langevin(dt=0.001, temperature=300.0, friction=1.0), 20, rng=np.random.default_rng(1))
        out[key] = (s.coords.copy(), s.velocities.copy(), s.stats()["graph_mode"], s)
    print({k: v[2] for k, v in out.items()})
    assert out["graph"][2] == 1 and out["stream"][2] == 0
    for k in ("stream", "logged"):
        assert np.array_equal(out["graph"][0], out[k][0]) and np.array_equal(out["graph"][1], out[k][1]), k
    monkeypatch.setenv("MOLLYB200_NO_GRAPH", "0")
    logged = out["logged"][3]
    assert len(logged.loggers["pe"].history) == 5
    for e_log, x_log in zip(logged.loggers["pe"].history, logged.loggers["x"].history):
        probe = _gb_dyn(g, dtype)
        probe.coords = np.asarray(x_log).astype(dtype)
        e = mb.potential_energy(probe)
        assert abs(e - e_log) <= H.etol(dtype, e), (e, e_log)
    # New GB parameters on a live context whose step graph has been captured: the next run must use them, as a fresh
    # context does (a step graph kept across mb_set_implicit_solvent would replay the old parameters). The all-pairs path
    # keeps the atoms in their original order in both contexts, so the two runs add in the same order.
    lang = mb.Langevin(dt=0.001, temperature=300.0, friction=1.0)
    s = _gb_dyn(g, dtype, brick=False)
    mb.simulate(s, lang, 10, rng=np.random.default_rng(4))
    assert s.stats()["graph_mode"] == 1
    x_mid, v_mid = s.coords.copy(), s.velocities.copy()
    gb2, _ = _inter(g, "gbn2", kappa=0.0, dist_cutoff=2.0)
    s.general_inters = (gb2,)
    s._set_implicit_solvent(gb2)
    mb.simulate(s, lang, 10, init_step=10, rng=np.random.default_rng(5))
    fresh = _gb_dyn(g, dtype, brick=False, kappa=0.0, dist_cutoff=2.0)
    fresh.coords, fresh.velocities = x_mid.copy(), v_mid.copy()
    mb.simulate(fresh, lang, 10, init_step=10, rng=np.random.default_rng(5))
    assert s.stats()["graph_mode"] == 1 and fresh.stats()["graph_mode"] == 1
    assert np.array_equal(s.coords, fresh.coords) and np.array_equal(s.velocities, fresh.velocities)
    # and the old parameters give a different trajectory (the comparison above can tell them apart)
    old = _gb_dyn(g, dtype, brick=False)
    old.coords, old.velocities = x_mid.copy(), v_mid.copy()
    mb.simulate(old, lang, 10, init_step=10, rng=np.random.default_rng(5))
    assert not np.array_equal(old.coords, fresh.coords)


def test_engine_refusals(g):
    s = _full_system(g, "obc2", F64)
    mb.forces(s)
    L, ctx = s._L, s._ctx
    n = s.n
    good = [np.full(n, 0.15), np.full(n, 0.12), np.ones(n), np.full(n, 0.8), np.full(n, 4.85)]

    def call(p, arrays=good, cls=None, d0=None, m0=None):
        arrs = [np.ascontiguousarray(a, np.float64) for a in arrays]
        return L.mb_set_implicit_solvent(ctx, C.byref(p), *[a.ctypes.data for a in arrs],
                                         None if cls is None else cls.ctypes.data, None if d0 is None else d0.ctypes.data,
                                         None if m0 is None else m0.ctypes.data)

    def params(**kw):
        base = dict(dist_cutoff=0.0, offset=0.009, probe_radius=0.14, sa_factor=28.39, factor_solute=-138.9,
                    factor_solvent=1.77, kappa=0.0, neck_scale=0.8, neck_cut=0.68, use_ace=1, n_neck_classes=0)
        base.update(kw)
        return mb.capi.MBGbsa(**base)
    assert call(params()) == mb.capi.MB_OK
    bad = [params(kappa=float("nan")), params(dist_cutoff=-1.0), params(offset=-0.1), params(n_neck_classes=33),
           params(sa_factor=float("inf"))]
    for p in bad:
        assert call(p) == mb.capi.MB_ERR_INVALID, p
    r0 = [np.full(n, 0.0)] + good[1:]
    assert call(params(), r0) == mb.capi.MB_ERR_INVALID
    rnan = good[:2] + [np.full(n, np.nan)] + good[3:]
    assert call(params(), rnan) == mb.capi.MB_ERR_INVALID
    cls = np.zeros(n, np.int32)
    cls[5] = 2
    tab = np.full(4, 0.27)
    assert call(params(n_neck_classes=2), good, cls, tab, tab) == mb.capi.MB_ERR_INVALID
    cls[5] = 1
    assert call(params(n_neck_classes=2), good, cls, tab, tab) == mb.capi.MB_OK
    neg = good[:1] + [np.full(n, -0.1)] + good[2:]  # a negative scaled radius (GBN2's sulphur screen) is allowed
    assert call(params(), neg) == mb.capi.MB_OK
    # atoms not set
    ctx2 = C.c_void_p()
    assert L.mb_ctx_create(0, 64, None, C.byref(ctx2)) == mb.capi.MB_OK
    try:
        arrs = [np.ascontiguousarray(a) for a in good]
        assert L.mb_set_implicit_solvent(ctx2, C.byref(params()), *[a.ctypes.data for a in arrs], None, None, None) == mb.capi.MB_ERR_STATE
    finally:
        L.mb_ctx_destroy(ctx2)
    with pytest.raises(NotImplementedError):
        mb.forces_virial(s)
    with pytest.raises(TypeError, match="implicit solvent"):
        mb.simulate(s, mb.MTSIntegrator(0.002, pi_fractions=(1, 1), si_fractions=(1, 1, 1), gi_fractions=(2,)), 2)
