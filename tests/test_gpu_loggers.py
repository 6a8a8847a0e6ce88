"""Device-side loggers (mb_simulate_vv_log): PotentialEnergy / KineticEnergy / TotalEnergy / Temperature / Coordinates /
Velocities loggers recorded inside one simulate call, against unlogged runs stopped at the logged steps and against the
reference's 6mrr pins (test/protein.jl:277-299)."""
import ctypes as C

import numpy as np
import pytest

import mbhelpers as H
import mollyb200 as mb
from test_gpu_parity import _pos_err

pytestmark = pytest.mark.gpu

F32, F64 = np.float32, np.float64


def _all_loggers(e=5, x=7):
    return {"pe": mb.PotentialEnergyLogger(e), "ke": mb.KineticEnergyLogger(e), "tot": mb.TotalEnergyLogger(e),
            "temp": mb.TemperatureLogger(e), "x": mb.CoordinatesLogger(x), "v": mb.VelocitiesLogger(x)}


def _lj(r_list):
    return (mb.LennardJones(cutoff=mb.ShiftedForceCutoff(1.0), use_neighbors=r_list > 0),)


def _fluid(dtype, r_list=1.2, loggers=None, cells=8):
    """2 048 argon atoms in a 4.6 nm box: the cell-list path with r_list > 0, the all-pairs path with r_list = 0."""
    s = H.make_system(H.lj_fluid(cells, dtype=dtype), _lj(r_list), dtype, r_list=r_list)
    s.loggers = dict(loggers or {})
    return s


def _sim(kind):
    if kind == "andersen":
        return mb.VelocityVerlet(dt=0.002, coupling=mb.AndersenThermostat(90.0, 0.05))
    if kind == "stream":
        return mb.VelocityVerlet(dt=0.002, remove_CM_motion=2)
    return mb.VelocityVerlet(dt=0.002)


OBSERVER_CASES = [("f32-brick", F32, 1.2, "plain"), ("f64-brick", F64, 1.2, "plain"), ("f64-allpairs", F64, 0.0, "plain"),
                  ("f64-stream", F64, 1.2, "stream"), ("f32-andersen", F32, 1.2, "andersen"),
                  ("f64-allpairs-andersen-stream", F64, 0.0, "andersen-stream")]


@pytest.mark.parametrize("name,dtype,r_list,kind", OBSERVER_CASES, ids=[c[0] for c in OBSERVER_CASES])
def test_logging_does_not_change_the_trajectory(name, dtype, r_list, kind):
    """Energies every 5 steps, frames every 7: coordinates and velocities are bit-identical to the unlogged run."""
    sim = _sim(kind.split("-")[0])
    if kind.endswith("stream"):
        sim.remove_CM_motion = 2
    out = []
    for loggers in (None, _all_loggers()):
        s = _fluid(dtype, r_list, loggers)
        mb.simulate(s, sim, 30, rng=np.random.default_rng(5))
        out.append((s.coords.copy(), s.velocities.copy(), s.stats()["graph_mode"]))
        if loggers:
            assert len(s.loggers["pe"].history) == 7 and len(s.loggers["x"].history) == 5
        s.close()
    (x0, v0, g0), (x1, v1, g1) = out
    print(f"[observer {name}] graph_mode unlogged={g0} logged={g1}")
    assert g0 == g1 == (0 if "stream" in kind else 1)
    assert np.array_equal(x0, x1) and np.array_equal(v0, v1)


def test_logging_with_bonded_terms_keeps_the_trajectory(golden_6mrr):
    """6mrr (bonded forces are added with float atomics, so runs agree to the f64 bar of the bonded VV test)."""
    g = golden_6mrr
    res = []
    for loggers in (None, _all_loggers(5, 7)):
        s = H.sixmrr_system({k: v.copy() for k, v in g.items()}, F64, r_list=1.2, n_steps=10)
        s.loggers = dict(loggers or {})
        mb.simulate(s, mb.VelocityVerlet(dt=0.0005), 20)
        res.append((s.coords.copy(), s.velocities.copy()))
        s.close()
    ex, ev = _pos_err(res[0][0], res[1][0], H.sixmrr_description(g)["box"]), np.abs(res[0][1] - res[1][1]).max()
    print(f"[observer 6mrr bonded] dx={ex:.3e} dv={ev:.3e}")
    assert ex < 1e-9 and ev < 1e-6


VALUE_CASES = [("f64-brick", F64, 1.2, "plain"), ("f32-brick", F32, 1.2, "plain"), ("f64-andersen", F64, 1.2, "andersen"),
               ("f64-allpairs-stream", F64, 0.0, "stream")]


@pytest.mark.parametrize("name,dtype,r_list,kind", VALUE_CASES, ids=[c[0] for c in VALUE_CASES])
def test_records_match_unlogged_runs_stopped_at_each_step(name, dtype, r_list, kind):
    n = 12
    s = _fluid(dtype, r_list, _all_loggers(3, 4))
    sim = _sim(kind)
    mb.simulate(s, sim, n, rng=np.random.default_rng(9))
    L = s.loggers
    e_steps, f_steps = mb.record_steps(3, n), mb.record_steps(4, n)
    assert e_steps == [0, 3, 6, 9, 12] and f_steps == [0, 4, 8, 12]
    assert [len(L[k].history) for k in ("pe", "ke", "tot", "temp", "x", "v")] == [5, 5, 5, 5, 4, 4]
    box = s.boundary.side_lengths
    worst = dict(pe=0.0, ke=0.0, x=0.0)
    for step in sorted(set(e_steps) | set(f_steps)):
        r = _fluid(dtype, r_list)
        mb.simulate(r, sim, step, rng=np.random.default_rng(9))
        if step in e_steps:
            k = e_steps.index(step)
            pe, ke = mb.potential_energy(r), mb.kinetic_energy(r)
            bar = (lambda e: 1e-9 * abs(e)) if dtype == F64 else (lambda e: H.etol(dtype, e))
            assert abs(L["pe"].history[k] - pe) <= bar(pe), (step, L["pe"].history[k], pe)
            assert abs(L["ke"].history[k] - ke) <= bar(ke), (step, L["ke"].history[k], ke)
            assert abs(L["tot"].history[k] - (pe + ke)) <= bar(pe) + bar(ke)
            assert abs(L["temp"].history[k] - mb.temperature(r)) <= 1e-9 * mb.temperature(r) + bar(ke) / ke * mb.temperature(r)
            worst["pe"] = max(worst["pe"], abs(L["pe"].history[k] - pe) / abs(pe))
            worst["ke"] = max(worst["ke"], abs(L["ke"].history[k] - ke) / ke)
        if step in f_steps:
            k = f_steps.index(step)
            assert np.array_equal(L["v"].history[k], r.velocities), step
            d = _pos_err(L["x"].history[k], r.coords, box)
            worst["x"] = max(worst["x"], d)
            assert d < (1e-12 if dtype == F64 else 1e-5) and (L["x"].history[k] >= 0).all()
        r.close()
    print(f"[values {name}] worst relative |dPE|={worst['pe']:.2e} |dKE|={worst['ke']:.2e} max|dx| frames={worst['x']:.2e}")
    s.close()


def test_6mrr_pme_reference_pins(golden_6mrr):
    """The 100-step PME run of test_zz_gpu_pme.py with loggers (f64, stream path): first KE / total energy / temperature
    records and the step-100 frames against OpenMM (test/protein.jl:284-299). simulate! removes the centre-of-mass motion
    before it runs the loggers at init_step (src/simulators.jl:563, :575), so the first records are the pins (taken on the
    starting velocities) less the kinetic energy of the centre-of-mass motion, 1/2 |sum m v|^2 / sum m = 0.93 kJ/mol here."""
    g = golden_6mrr
    m = H.sixmrr_description(g)["mass"]
    p_cm = (m[:, None] * g["velocities_300K"]).sum(0)
    ke_cm = 0.5 * (p_cm @ p_cm) / m.sum()
    s = H.sixmrr_pme_system(g, F64, exact=True, velocities=g["velocities_300K"])
    s.loggers = {"ke": mb.KineticEnergyLogger(10), "tot": mb.TotalEnergyLogger(10), "temp": mb.TemperatureLogger(10),
                 "x": mb.CoordinatesLogger(100), "v": mb.VelocitiesLogger(100)}
    mb.simulate(s, mb.VelocityVerlet(dt=0.0005), 100)
    L = s.loggers
    ke0, e0, t0 = L["ke"].history[0], L["tot"].history[0], L["temp"].history[0]
    print(f"[6mrr PME loggers] KE0={ke0!r} E0={e0!r} T0={t0!r} graph_mode={s.stats()['graph_mode']}")
    assert s.stats()["graph_mode"] == 0
    assert abs(ke0 + ke_cm - 65521.87288132431) < 1.5e-8 * 65521.87288132431
    assert abs(e0 + ke_cm - 96522.24858589929) < 1.5e-8 * 96522.24858589929
    assert abs(t0 * (ke0 + ke_cm) / ke0 - 329.3202932884933) < 1.5e-8 * 329.3202932884933
    assert len(L["x"].history) == 2 and len(L["ke"].history) == 11
    box = g["box"]
    x_ref = g["coordinates_100steps"] - np.floor(g["coordinates_100steps"] / box) * box
    dx = _pos_err(L["x"].history[-1], x_ref, box)
    dv = np.linalg.norm(L["v"].history[-1] - g["velocities_100steps"], axis=1).max()
    print(f"[6mrr PME loggers] step-100 frames: max|dx|={dx:.3e} (bar 1e-10) max|dv|={dv:.3e} (bar 1e-7)")
    assert dx < 1e-10 and dv < 1e-7
    assert np.array_equal(L["x"].history[-1], s.coords) and np.array_equal(L["v"].history[-1], s.velocities)
    s.close()


@pytest.mark.parametrize("cut", ["distance", "shifted_potential", "shifted_force", "cubic_spline"])
def test_energy_conservation_in_one_call(cut):
    """The reference protocol of test_gpu_parity.py (test/energy_conservation.jl:9-75) as one 10 000-step call with
    TotalEnergyLogger(100): max |E - E0| < 5e-4 kJ/mol."""
    n, L, rc = 2000, 5.0, 3.0
    rng = np.random.default_rng(11)
    pts = np.empty((0, 3))
    while len(pts) < n:
        c = rng.random((4 * n, 3)) * L
        for q in c:
            d = pts - q
            d -= L * np.round(d / L)
            if len(pts) == 0 or (np.einsum("ij,ij->i", d, d) > 0.01).all():
                pts = np.vstack([pts, q])
                if len(pts) == n:
                    break
    cutoff = {"distance": mb.DistanceCutoff(rc), "shifted_potential": mb.ShiftedPotentialCutoff(rc),
              "shifted_force": mb.ShiftedForceCutoff(rc), "cubic_spline": mb.CubicSplineCutoff(rc, rc + 0.5)}[cut]
    atoms = mb.atoms_from_arrays(np.full(n, 40.0), np.zeros(n), np.full(n, 0.05), np.full(n, 0.2), np.float64)
    v = rng.normal(0.0, np.sqrt(mb.BOLTZMANN_K * 1.0 / 40.0), (n, 3))
    s = mb.System(atoms=atoms, coords=pts.copy(), boundary=mb.CubicBoundary(L), velocities=v,
                  pairwise_inters=(mb.LennardJones(cutoff=cutoff, use_neighbors=True),),
                  neighbor_finder=mb.GPUNeighborFinder(dist_cutoff=rc + (0.5 if cut == "cubic_spline" else 0.0)), dtype=np.float64,
                  loggers={"e": mb.TotalEnergyLogger(100)})
    mb.simulate(s, mb.VelocityVerlet(dt=0.001, remove_CM_motion=0), 10_000)
    e = np.array(s.loggers["e"].history)
    worst = np.abs(e - e[0]).max()
    print(f"[energy conservation in one call, {cut}] records={len(e)} E0={e[0]:.6f} max|E-E0|={worst:.3e} kJ/mol (bar 5e-4)")
    assert len(e) == 101 and worst < 5e-4
    s.close()


# ---------------------------------------------------------------------------------------------------
# bookkeeping
# ---------------------------------------------------------------------------------------------------
def _small(dtype=F64, loggers=None):
    return _fluid(dtype, 1.2, loggers, cells=6)


@pytest.mark.parametrize("run_loggers,count", [(True, 7), (False, 0), ("skipstart", 6)])
def test_run_loggers(run_loggers, count):
    s = _small(loggers={"x": mb.CoordinatesLogger(1), "e": mb.PotentialEnergyLogger(2)})
    x0 = s.coords.copy()
    mb.simulate(s, mb.VelocityVerlet(dt=0.002), 6, run_loggers=run_loggers)
    assert len(s.loggers["x"].history) == count
    assert len(s.loggers["e"].history) == {7: 4, 0: 0, 6: 3}[count]
    if count:
        first = s.loggers["x"].history[0]
        assert (np.abs(first - x0).max() < 1e-12) == (run_loggers is True)
        assert np.array_equal(s.loggers["x"].history[-1], s.coords)
    s.close()


def test_init_step_and_intervals_not_dividing_n_steps():
    s = _small(loggers={"a": mb.KineticEnergyLogger(3), "b": mb.KineticEnergyLogger(5), "x": mb.CoordinatesLogger(4),
                        "v": mb.VelocitiesLogger(6)})
    mb.simulate(s, mb.VelocityVerlet(dt=0.002), 13, init_step=3)
    lens = {k: len(lg.history) for k, lg in s.loggers.items()}
    assert lens == {"a": 5, "b": 3, "x": 4, "v": 2}, lens  # a: 3 (init_step), 6, 9, 12, 15; b: 5, 10, 15; x: 4, 8, 12, 16; v: 6, 12
    s.close()


@pytest.mark.parametrize("pair", [(3, 5), (4, 6)])
def test_each_logger_keeps_its_own_steps(pair):
    """Loggers of different intervals in one run give what each gives alone (the engine records at their gcd)."""
    a, b = pair
    both = _small(loggers={"pa": mb.PotentialEnergyLogger(a), "kb": mb.KineticEnergyLogger(b), "xa": mb.CoordinatesLogger(a),
                           "vb": mb.VelocitiesLogger(b)})
    mb.simulate(both, mb.VelocityVerlet(dt=0.002), 20)
    for name, lg in (("pa", mb.PotentialEnergyLogger(a)), ("kb", mb.KineticEnergyLogger(b)), ("xa", mb.CoordinatesLogger(a)),
                     ("vb", mb.VelocitiesLogger(b))):
        alone = _small(loggers={name: lg})
        mb.simulate(alone, mb.VelocityVerlet(dt=0.002), 20)
        h0, h1 = both.loggers[name].history, alone.loggers[name].history
        assert len(h0) == len(h1) == len(mb.record_steps(lg.n_steps, 20))
        assert all(np.array_equal(p, q) for p, q in zip(h0, h1)), name
        alone.close()
    both.close()


def test_consecutive_calls_equal_one_long_call():
    one = _small(loggers={"e": mb.TotalEnergyLogger(5), "x": mb.CoordinatesLogger(10)})
    mb.simulate(one, mb.VelocityVerlet(dt=0.002), 30)
    two = _small(loggers={"e": mb.TotalEnergyLogger(5), "x": mb.CoordinatesLogger(10)})
    mb.simulate(two, mb.VelocityVerlet(dt=0.002), 10)
    mb.simulate(two, mb.VelocityVerlet(dt=0.002), 20, init_step=10, run_loggers="skipstart")
    e1, e2 = np.array(one.loggers["e"].history), np.array(two.loggers["e"].history)
    assert len(e1) == len(e2) == 7 and len(two.loggers["x"].history) == 4
    print(f"[consecutive calls] max|dE|={np.abs(e1 - e2).max():.3e}")
    assert np.abs(e1 - e2).max() < 1e-9 * np.abs(e1).max()
    for p, q in zip(one.loggers["x"].history, two.loggers["x"].history):
        assert _pos_err(p, q, one.boundary.side_lengths) < 1e-9
    one.close(), two.close()


def test_fewer_than_four_steps_run_without_the_graph():
    s = _small(loggers=_all_loggers(1, 1))
    mb.simulate(s, mb.VelocityVerlet(dt=0.002), 3)
    assert s.stats()["graph_mode"] == 0
    assert len(s.loggers["pe"].history) == 4 and len(s.loggers["v"].history) == 4
    assert np.array_equal(s.loggers["x"].history[-1], s.coords) and np.array_equal(s.loggers["v"].history[-1], s.velocities)
    s.close()


def test_triclinic_boundary():
    rng = np.random.default_rng(3)
    n, L = 64, 2.2
    bnd = mb.TriclinicBoundary([L, 0.0, 0.0], [0.4, L, 0.0], [-0.3, 0.5, L])
    grid = np.stack(np.meshgrid(*[np.arange(4)] * 3, indexing="ij"), -1).reshape(-1, 3) / 4.0
    x = grid @ bnd.basis_vectors + rng.normal(0, 0.01, (n, 3))
    v = rng.normal(0, 0.2, (n, 3))
    atoms = mb.atoms_from_arrays(np.full(n, 40.0), np.zeros(n), np.full(n, 0.34), np.full(n, 0.5), F64)
    res = []
    for loggers in (None, _all_loggers(2, 3)):
        s = mb.System(atoms=atoms, coords=x.copy(), boundary=bnd, velocities=v.copy(),
                      pairwise_inters=(mb.LennardJones(cutoff=mb.ShiftedForceCutoff(0.8)),), dtype=F64, loggers=loggers)
        mb.simulate(s, mb.VelocityVerlet(dt=0.002), 12)
        res.append(s)
    assert np.array_equal(res[0].coords, res[1].coords) and np.array_equal(res[0].velocities, res[1].velocities)
    L_ = res[1].loggers
    assert len(L_["pe"].history) == 7 and len(L_["x"].history) == 5
    assert np.array_equal(L_["x"].history[-1], res[1].coords) and np.array_equal(L_["v"].history[-1], res[1].velocities)
    assert abs(L_["pe"].history[-1] - mb.potential_energy(res[1])) < 1e-9 * abs(L_["pe"].history[-1])
    for s in res:
        s.close()


def test_torch_device_state():
    torch = pytest.importorskip("torch")
    sd = H.lj_fluid(6, dtype=F32)
    host = H.make_system(sd, _lj(1.2), F32, r_list=1.2)
    host.loggers = _all_loggers(3, 4)
    mb.simulate(host, mb.VelocityVerlet(dt=0.002), 12)
    dev = H.make_system(sd, _lj(1.2), F32, r_list=1.2)
    dev.coords = torch.from_numpy(sd["coords"].copy()).cuda()
    dev.velocities = torch.from_numpy(sd["velocities"].copy()).cuda()
    dev.loggers = _all_loggers(3, 4)
    mb.simulate(dev, mb.VelocityVerlet(dt=0.002), 12)
    for k in host.loggers:
        hh, dh = host.loggers[k].history, dev.loggers[k].history
        assert len(hh) == len(dh) > 0
        assert all(isinstance(t, torch.Tensor) and t.is_cuda for t in dh)
        for a, b in zip(hh, dh):
            assert np.array_equal(np.asarray(a), b.cpu().numpy()), k
    host.close(), dev.close()


def test_c_abi_refuses_bad_log_descriptors():
    s = _small()
    ctx = s.engine()
    L = s._L
    p = mb.capi.MBVVParams()
    p.dt, p.n_steps, p.init_step, p.remove_cm_every = 0.002, 10, 0, 1
    e = np.zeros((3, 3))
    frames = np.zeros((3, s.n, 3))

    def call(**kw):
        d = mb.capi.MBLog()
        for k, v in kw.items():
            setattr(d, k, v)
        return L.mb_simulate_vv_log(ctx, s.coords.ctypes.data, s.velocities.ctypes.data, C.byref(p), C.byref(d))

    x0 = s.coords.copy()
    # energies every 5 with log_initial: steps 0, 5, 10 -> 3 records fit, 2 do not
    assert call(energy_every=5, log_initial=1, energies=e.ctypes.data, energy_capacity=2) == mb.capi.MB_ERR_INVALID
    assert "capacity" in L.mb_last_error().decode()
    assert call(energy_every=5, log_initial=1, energy_capacity=3) == mb.capi.MB_ERR_INVALID  # null output
    assert call(coords_every=4, coords_capacity=3) == mb.capi.MB_ERR_INVALID
    assert call(vels_every=-1) == mb.capi.MB_ERR_INVALID
    assert np.array_equal(s.coords, x0)  # refused before any work
    d = mb.capi.MBLog()
    d.energy_every, d.log_initial, d.energies, d.energy_capacity = 5, 1, e.ctypes.data, 3
    d.coords_every, d.coords, d.coords_capacity = 4, frames.ctypes.data, 3
    assert L.mb_simulate_vv_log(ctx, s.coords.ctypes.data, s.velocities.ctypes.data, C.byref(p), C.byref(d)) == 0
    assert (d.n_energies, d.n_coords, d.n_vels) == (3, 3, 0)
    assert list(e[:, 0]) == [0.0, 5.0, 10.0]
    s.close()


def test_droplet_overflow_retry_keeps_exact_records():
    """The drifting droplet of test_gpu_celllist_edges.py overflows the first capacities; simulate retries, and the
    histories hold each step exactly once."""
    side, radius = 12.0, 3.5
    box = np.array([side] * 3)
    sd = H.argon_droplet(radius, box, [side - 1.5 - radius, side / 2, side / 2], seed=11)
    sd["velocities"] = sd["velocities"] + np.array([12.0, 0.0, 0.0])
    inters = (mb.LennardJones(cutoff=mb.ShiftedForceCutoff(1.2), use_neighbors=True),)
    s = H.make_system(sd, inters, F64, r_list=1.3)
    s.loggers = {"e": mb.PotentialEnergyLogger(10), "x": mb.CoordinatesLogger(50), "v": mb.VelocitiesLogger(50)}
    mb.simulate(s, mb.VelocityVerlet(dt=0.002, remove_CM_motion=0), 200)
    st = s.stats()
    pe = np.array(s.loggers["e"].history)
    print(f"[droplet overflow with loggers] records={len(pe)} frames={len(s.loggers['x'].history)} rebuilds={st['n_rebuilds']}")
    assert len(pe) == 21 and len(s.loggers["x"].history) == 5 and len(s.loggers["v"].history) == 5
    assert len(np.unique(pe)) == 21
    assert np.array_equal(s.loggers["x"].history[-1], s.coords) and np.array_equal(s.loggers["v"].history[-1], s.velocities)
    s.close()
