"""CPU tests of the generalized-Born oracle (tests/gbsa_oracle.py) and of the implicit-solvent Python layer: the reference's
"Implicit solvent" check (test/protein.jl:663-707) against OpenMM's obc2/gbn2 forces and energies on 6mrr without water,
GB forces against central finite differences of the GB energy, the C-ABI parameter layout against the header, and the
refusals the Python layer makes before any GPU work."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import gbsa_oracle as gbo
import mbhelpers as H
import mollyb200 as mb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def g():
    return np.load(os.path.join(ROOT, "tests", "golden", "6mrr_gb.npz"))


def pair_forces_energy(g, x):
    """LennardJones + Coulomb with DistanceCutoff(5 nm) over all pairs, exclusions skipped, 1-4 pairs scaled (what
    System(...; nonbonded_method=:none, dist_cutoff=5 nm) builds), f64."""
    n = len(x)
    d = x[None, :, :] - x[:, None, :]
    r2 = np.einsum("ijk,ijk->ij", d, d)
    w_lj, w_c = np.ones((n, n)), np.ones((n, n))
    ex, sp = g["excluded"], g["special"]
    for w in (w_lj, w_c):
        w[ex[:, 0], ex[:, 1]] = w[ex[:, 1], ex[:, 0]] = 0
        np.fill_diagonal(w, 0)
    w_lj[sp[:, 0], sp[:, 1]] = w_lj[sp[:, 1], sp[:, 0]] = float(g["lj14scale"])
    w_c[sp[:, 0], sp[:, 1]] = w_c[sp[:, 1], sp[:, 0]] = float(g["coulomb14scale"])
    inside = r2 <= float(g["dist_cutoff"]) ** 2
    w_lj, w_c = w_lj * inside, w_c * inside
    r2s = np.where(w_c + w_lj > 0, r2, 1.0)
    sig = (g["sigma"][:, None] + g["sigma"][None, :]) / 2
    eps = np.sqrt(g["eps"][:, None] * g["eps"][None, :])
    s6 = (sig * sig / r2s) ** 3
    e_lj = 4 * eps * (s6 * s6 - s6) * w_lj
    f_lj = 24 * eps * (2 * s6 * s6 - s6) / r2s * w_lj  # -dE/dr / r
    qq = gbo.COULOMB_CONST * g["charge"][:, None] * g["charge"][None, :]
    r = np.sqrt(r2s)
    e_c = qq / r * w_c
    f_c = qq / (r2s * r) * w_c
    f = -np.einsum("ijk,ij->ik", d, f_lj + f_c)
    return f, 0.5 * float(np.sum(e_lj + e_c))


@pytest.mark.parametrize("model", ["obc2", "gbn2"])
def test_openmm_goldens(g, model):
    x = g["coords"]
    p = gbo.from_golden(g, model)
    f_gb, e_gb = gbo.forces_energy(x, g["charge"], p, box=g["box"])
    f_pair, e_pair = pair_forces_energy(g, x)
    f_b, e_b = H.bonded_forces_oracle(g, x)
    df = np.linalg.norm(f_gb + f_pair + f_b - g[f"forces_{model}"], axis=1).max()
    de = abs(e_gb + e_pair + e_b - float(g[f"energy_{model}"]))
    print(f"[{model}] max |dF| = {df:.2e} kJ/mol/nm, |dE| = {de:.2e} kJ/mol")
    assert df < 1e-3 and de < 1e-2  # the reference's bars (test/protein.jl:688, :694)


def _cluster(g, n=60, seed=0):
    """The n atoms nearest the protein's first atom: a dense, charged piece of the fixture for finite differences."""
    x = g["coords"]
    idx = np.argsort(np.linalg.norm(x - x[0], axis=1), kind="stable")[:n]
    rng = np.random.default_rng(seed)
    return idx, x[idx] + rng.normal(0, 0.01, (n, 3))


def _sub(p, idx):
    kw = {k: getattr(p, k) for k in p.__dataclass_fields__}
    for k in ("offset_radii", "scaled_offset_radii", "alpha", "beta", "gamma"):
        kw[k] = np.asarray(kw[k])[idx]
    if p.has_neck:
        kw["neck_class"] = np.asarray(p.neck_class)[idx]
    return gbo.GB(**kw)


@pytest.mark.parametrize("model", ["obc2", "gbn2"])
@pytest.mark.parametrize("kappa", [0.0, 1.0])
def test_forces_are_minus_energy_gradient(g, model, kappa):
    idx, x = _cluster(g)
    p = _sub(gbo.from_golden(g, model, kappa=kappa), idx)
    q = g["charge"][idx]
    f, _ = gbo.forces_energy(x, q, p)
    h = 1e-6
    fd = np.zeros_like(x)
    for i in range(len(x)):
        for k in range(3):
            xp, xm = x.copy(), x.copy()
            xp[i, k] += h
            xm[i, k] -= h
            fd[i, k] = -(gbo.energy(xp, q, p) - gbo.energy(xm, q, p)) / (2 * h)
    err = np.abs(f - fd).max()
    print(f"[{model} kappa={kappa}] max |F + dE/dx| = {err:.2e} (max |F| {np.abs(f).max():.1f})")
    assert err < 1e-5 * max(1.0, np.abs(f).max())


def test_triclinic_minimum_image_matches_rectangular_for_a_rectangular_basis(g):
    from oracle.triclinic import Triclinic
    idx, x = _cluster(g, 40)
    p = _sub(gbo.from_golden(g, "gbn2", dist_cutoff=1.2), idx)
    box = np.array([2.0, 2.1, 2.2])
    x = x - np.floor(x / box) * box
    f1, e1 = gbo.forces_energy(x, g["charge"][idx], p, box=box)
    f2, e2 = gbo.forces_energy(x, g["charge"][idx], p, tric=Triclinic(np.diag(box)))
    assert np.abs(f1 - f2).max() < 1e-9 and abs(e1 - e2) < 1e-9


def test_gbsa_params_layout_matches_header(tmp_path):
    P = mb.capi.MBGbsa
    assert mb.capi.MB_GB_MAX_NECK_CLASSES == 32 and C.sizeof(P) == 80
    src = tmp_path / "t.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "mollyb200.h"\nint main(void) {\n'
                   '    printf("%zu %zu %zu %d\\n", sizeof(mb_gbsa_t), offsetof(mb_gbsa_t, use_ace), '
                   'offsetof(mb_gbsa_t, n_neck_classes), MB_GB_MAX_NECK_CLASSES);\n    return 0;\n}\n')
    exe = tmp_path / "t"
    subprocess.run(["cc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()
    assert out == [str(C.sizeof(P)), str(P.use_ace.offset), str(P.n_neck_classes.offset), "32"]


def test_exported():
    assert "mb_set_implicit_solvent" in mb.capi.EXPORTED
    L = mb.capi.load()
    assert L.mb_set_implicit_solvent(None, None, None, None, None, None, None, None, None, None) == mb.capi.MB_ERR_INVALID
    assert b"null context" in L.mb_last_error()


def _gb(model="gbn2", n=4, **kw):
    base = dict(offset_radii=np.full(n, 0.15), scaled_offset_radii=np.full(n, 0.12), alpha=np.ones(n), beta=np.full(n, 0.8),
                gamma=np.full(n, 4.85))
    if model == "gbn2":
        base.update(neck_class=np.zeros(n, np.int32), d0=np.full((1, 1), 2.7), m0=np.full((1, 1), 0.01))
        base.update(kw)
        return mb.ImplicitSolventGBN2(**base)
    base.update(kw)
    return mb.ImplicitSolventOBC(**base)


def test_python_refusals():
    with pytest.raises(ValueError):
        _gb(offset_radii=np.full(3, 0.15))  # length mismatch
    with pytest.raises(ValueError):
        _gb(neck_class=np.array([0, 1, 0, 0], np.int32))  # class outside the table
    with pytest.raises(ValueError):
        _gb(d0=np.zeros((1, 2)))
    gb = _gb()
    s = mb.System(atoms=mb.atoms_from_arrays(np.ones(4), np.zeros(4), np.zeros(4), np.zeros(4), np.float64),
                  coords=np.random.default_rng(0).random((4, 3)), boundary=mb.CubicBoundary(3.0), general_inters=(gb,),
                  dtype=np.float64)
    with pytest.raises(NotImplementedError):
        mb.forces_virial(s)
    s.general_inters = (gb, mb.LJDispersionCorrection(1.0))
    mb.mts_levels(s, mb.MTSIntegrator(0.002, gi_fractions=(1, 2)))
    with pytest.raises(TypeError, match="implicit solvent"):
        mb.mts_levels(s, mb.MTSIntegrator(0.002, gi_fractions=(2, 1)))
