"""csrc/cutoffs2.cuh (CubicSplineCutoff / PolynomialCutoff, SURVEY.md §8(f)-4) compiled for the HOST and checked against
the reference's literals (test/interactions.jl:1574-1603) and the C oracle. The GPU counterpart is tests/test_gpu_parity.py::test_two_point_cutoffs_*."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import oracle as o

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def hostlib(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out = str(tmp_path_factory.mktemp("cut2h") / "libcut2h.so")
    p = subprocess.run([nvcc, "-std=c++17", "-O2", "-shared", "-Xcompiler", "-fPIC", "-ccbin", "/usr/bin/g++", "-gencode",
                        "arch=compute_90a,code=sm_90a", "-o", out, os.path.join(ROOT, "tests", "host", "cutoffs_host.cu")],
                       capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-3000:]
    return C.CDLL(out)


def _lj(lib, kind, ra, rc, sigma, eps, r):
    fr, e = C.c_double(), C.c_double()
    lib.cut2h_lj(kind, C.c_double(ra), C.c_double(rc), C.c_double(sigma), C.c_double(eps), C.c_double(r), C.byref(fr), C.byref(e))
    return fr.value, e.value


def test_two_point_cutoffs_on_host(hostlib):
    # the reference's literals: sigma 0.3, eps 0.2, r = 0.7, dist_act 0.6, dist_cut 0.8; its force(...)[1] is f with fs[i] -= f
    for kind, f_ref, e_ref in ((4, -0.06201171875, -0.00312500000), (5, -0.06716652806, -0.00246320097)):
        fr, e = _lj(hostlib, kind, 0.6, 0.8, 0.3, 0.2, 0.7)
        assert abs(fr * 0.7 - f_ref) < 1e-9 and abs(e - e_ref) < 1e-9  # F = (F/r) r; negative = attractive
    # against the C oracle over the whole range (below r_act: plain LJ; beyond r_cut the caller zeroes)
    rng = np.random.default_rng(3)
    for kind, okind in ((4, o.CUT_CUBIC_SPLINE), (5, o.CUT_POLYNOMIAL)):
        for _ in range(200):
            sigma, eps = rng.uniform(0.25, 0.4), rng.uniform(0.1, 1.0)
            ra = rng.uniform(0.5, 0.9)
            rc = ra + rng.uniform(0.05, 0.4)
            r = rng.uniform(0.3, rc)
            s = o.OracleSystem(box=np.array([6.0, 6.0, 6.0]), mass=np.ones(2), charge=np.zeros(2), sigma=np.full(2, sigma),
                               eps=np.full(2, eps), inters=[o.Inter(o.LJ, okind, rc, r_act=ra)])
            f, e_ref, _ = s.forces_allpairs(np.array([[1.0, 1.0, 1.0], [1.0 + r, 1.0, 1.0]]))
            fr, e = _lj(hostlib, kind, ra, rc, sigma, eps, r)
            assert abs(fr * r - f[1, 0]) < 1e-9 * max(1.0, abs(f[1, 0]))  # the oracle's force on atom j along +x is F
            assert abs(e - e_ref) < 1e-10 * max(1.0, abs(e_ref))
    # continuity at both ends (what the cutoffs are for): V and F continuous at r_act, both zero at r_cut
    for kind in (4, 5):
        ra, rc = 0.6, 0.8
        below, above = _lj(hostlib, kind, ra, rc, 0.3, 0.2, ra - 1e-9), _lj(hostlib, kind, ra, rc, 0.3, 0.2, ra + 1e-9)
        assert abs(below[0] - above[0]) < 1e-6 and abs(below[1] - above[1]) < 1e-8
        end = _lj(hostlib, kind, ra, rc, 0.3, 0.2, rc)
        assert abs(end[0]) < 1e-12 and abs(end[1]) < 1e-12
    # Coulomb flavour: same switch on V = kqq / r, against the oracle's Coulomb branch over the whole range
    ke = 138.93545764
    for kind, okind in ((4, o.CUT_CUBIC_SPLINE), (5, o.CUT_POLYNOMIAL)):
        for _ in range(200):
            qi, qj = rng.uniform(-1, 1, 2)
            ra = rng.uniform(0.5, 0.9)
            rc = ra + rng.uniform(0.05, 0.4)
            r = rng.uniform(0.3, rc * 1.1)
            s = o.OracleSystem(box=np.array([6.0, 6.0, 6.0]), mass=np.ones(2), charge=np.array([qi, qj]), sigma=np.zeros(2),
                               eps=np.zeros(2), inters=[o.Inter(o.COULOMB, okind, rc, r_act=ra)])
            f, e_ref, _ = s.forces_allpairs(np.array([[1.0, 1.0, 1.0], [1.0 + r, 1.0, 1.0]]))
            fr, e = C.c_double(), C.c_double()
            hostlib.cut2h_coul(kind, C.c_double(ra), C.c_double(rc), C.c_double(ke * qi * qj), C.c_double(r), C.byref(fr), C.byref(e))
            frv, ev = (fr.value, e.value) if r <= rc else (0.0, 0.0)  # the caller applies the r <= r_c test
            assert abs(frv * r - f[1, 0]) < 1e-9 * max(1.0, abs(f[1, 0]))
            assert abs(ev - e_ref) < 1e-10 * max(1.0, abs(e_ref))
    # Coulomb flavour: same switch on V = kqq / r
    fr, e = C.c_double(), C.c_double()
    hostlib.cut2h_coul(5, C.c_double(0.6), C.c_double(0.8), C.c_double(138.93545764), C.c_double(0.8), C.byref(fr), C.byref(e))
    assert abs(fr.value) < 1e-10 and abs(e.value) < 1e-10
