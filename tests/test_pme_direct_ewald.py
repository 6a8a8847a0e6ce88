"""The PME checker (oracle/pme.py) against a direct reciprocal-space Ewald sum, on the CPU.

The device PME is compared with oracle/pme.py (tests/test_gpu_pme_matrix.py), and oracle/pme.py is pinned against OpenMM
only for 6mrr and the three waters (tests/test_oracle.py, tests/test_pme_host.py). This file closes the loop on the boxes,
meshes and charges of the GPU matrix: an explicit k-vector sum with exact structure factors, no mesh and no B-splines,
converged in k_max, is the quantity smooth PME approximates. Same alpha, same self and neutralising-background terms.

  E_recip = f / (2 pi V) sum_{m != 0} exp(-pi^2 m^2 / alpha^2) / m^2 |S(m)|^2,   S(m) = sum_j q_j exp(2 pi i m.r_j)
  F_i     = 2 f q_i / V sum_{m != 0} exp(-pi^2 m^2 / alpha^2) / m^2 m Im(conj(S(m)) exp(2 pi i m.r_i))

with m = (kx / Lx, ky / Ly, kz / Lz) and f = k_e / eps_r. PME's error is controlled by error_tol (the mesh and alpha both
follow from it); the bars below are the errors measured on these systems with about 5x headroom, and the error must
shrink as error_tol does."""
import numpy as np
import pytest

from oracle import pme

# box, r_cut, error_tol: the shapes of the GPU matrix (cubic, strongly anisotropic, K = 6 in x, a large fine mesh)
BOXES = {
    "cubic": np.array([3.0, 3.0, 3.0]),
    "aniso": np.array([2.0, 3.3, 5.1]),
    "k6": np.array([0.8, 1.0, 3.1]),
}


def charged_system(box, n, charges, seed):
    """Uniform random coordinates in the box and random charges: 'neutral', 'plus3' / 'minus3' (net charge +-3 e) or
    'zeros' (about 30 % of the atoms uncharged, the rest neutral)."""
    rng = np.random.default_rng(seed)
    x = rng.random((n, 3)) * box
    q = rng.normal(0.0, 0.5, n)
    if charges == "zeros":
        zero = rng.random(n) < 0.3
        q[~zero] -= q[~zero].mean()
        q[zero] = 0.0
    else:
        q -= q.mean()
        q += {"neutral": 0.0, "plus3": 3.0, "minus3": -3.0}[charges] / n
    return x, q


def direct_ewald(x, q, box, alpha, eps_r=1.0, m_cut_sigmas=6.5):
    """Reciprocal-space Ewald energy (incl. self and background terms) and forces by an explicit k-vector sum. Every m with
    pi^2 m^2 / alpha^2 <= m_cut_sigmas^2 is summed: exp(-42) ~ 6e-19 at the default, far below f64 resolution."""
    f = pme.COULOMB_CONST / eps_r
    V = float(np.prod(box))
    m_cut = m_cut_sigmas * alpha / np.pi
    kmax = [int(np.ceil(m_cut * L)) for L in box]
    ks = [np.arange(-k, k + 1) for k in kmax]
    ms = [k / L for k, L in zip(ks, box)]
    # per-dimension phase factors exp(2 pi i m_d x_d): (n, 2 kmax_d + 1)
    ph = [np.exp(2j * np.pi * np.outer(x[:, d], ms[d])) for d in range(3)]
    m2 = ms[0][:, None, None] ** 2 + ms[1][None, :, None] ** 2 + ms[2][None, None, :] ** 2
    with np.errstate(divide="ignore"):
        g = np.exp(-np.pi ** 2 * m2 / alpha ** 2) / m2
    g[kmax[0], kmax[1], kmax[2]] = 0.0
    g[np.pi ** 2 * m2 / alpha ** 2 > m_cut_sigmas ** 2] = 0.0
    S = np.einsum("j,ja,jb,jc->abc", q, ph[0], ph[1], ph[2], optimize=True)
    e_recip = f / (2.0 * np.pi * V) * float((g * (S.real ** 2 + S.imag ** 2)).sum())
    A = g * np.conj(S)
    F = np.empty_like(x)
    for d in range(3):
        w = [ph[0], ph[1], ph[2]]
        w[d] = w[d] * ms[d][None, :]
        F[:, d] = 2.0 * f / V * q * np.einsum("abc,ia,ib,ic->i", A, w[0], w[1], w[2], optimize=True).imag
    e_self = -f * alpha / np.sqrt(np.pi) * (q ** 2).sum() - f * np.pi * q.sum() ** 2 / (2.0 * V * alpha ** 2)
    return F, e_recip + e_self


def _errors(x, q, box, r_cut, tol, eps_r=1.0):
    alpha = pme.pme_alpha(r_cut, tol)
    f_ref, e_ref = direct_ewald(x, q, box, alpha, eps_r)
    f, e, _ = pme.pme_reciprocal(x, q, box, r_cut=r_cut, error_tol=tol, eps_r=eps_r)
    return np.abs(f - f_ref).max() / np.abs(f_ref).max(), abs(e - e_ref) / abs(e_ref)


def test_direct_ewald_is_converged_in_kmax():
    """The reference sum itself: widening the k-space sphere changes nothing beyond rounding (the energy, a difference of
    two terms of about 2000 kJ/mol here, is 4.4 kJ/mol; at 5.5 instead of 6.5 Gaussian widths it moves by 7e-12 of it)."""
    x, q = charged_system(BOXES["aniso"], 60, "plus3", seed=1)
    alpha = pme.pme_alpha(1.0, 1e-5)
    f1, e1 = direct_ewald(x, q, BOXES["aniso"], alpha)
    f2, e2 = direct_ewald(x, q, BOXES["aniso"], alpha, m_cut_sigmas=8.0)
    assert np.abs(f1 - f2).max() <= 1e-14 * np.abs(f2).max() and abs(e1 - e2) <= 1e-12 * abs(e2)


def test_direct_ewald_translation_and_charge_inversion():
    """Sanity of the reference sum: a rigid shift by lattice vectors and by an arbitrary vector leaves E and F unchanged,
    and flipping every charge leaves them unchanged too (E and F are quadratic in q); the forces of a neutral system sum
    to zero."""
    box = BOXES["cubic"]
    x, q = charged_system(box, 40, "neutral", seed=2)
    alpha = pme.pme_alpha(1.0, 5e-4)
    f0, e0 = direct_ewald(x, q, box, alpha)
    for xs in (x + box * np.array([1, -1, 2]), x + np.array([0.123, -0.77, 1.9])):
        f1, e1 = direct_ewald(xs, q, box, alpha)
        assert np.abs(f1 - f0).max() <= 1e-11 * np.abs(f0).max() and abs(e1 - e0) <= 1e-12 * abs(e0)
    f1, e1 = direct_ewald(x, -q, box, alpha)
    assert np.abs(f1 - f0).max() <= 1e-12 * np.abs(f0).max() and abs(e1 - e0) <= 1e-12 * abs(e0)
    assert np.abs(f0.sum(0)).max() <= 1e-11 * np.abs(f0).max()


# Measured max relative errors of oracle/pme.py against the direct sum on these systems (force: max|dF| / max|F|,
# energy: |dE| / |E|), worst over the boxes, charge sets and eps_r below: error_tol 1e-3 -> F 1.3e-3, E 2.3e-4;
# 5e-4 -> F 6.7e-4, E 1.1e-4; 1e-5 -> F 1.7e-5, E 1.1e-6. Bars: about 5x those.
BARS = {1e-3: (6.5e-3, 1.2e-3), 5e-4: (3.5e-3, 5.5e-4), 1e-5: (8.5e-5, 5.5e-6)}


@pytest.mark.parametrize("box_name", list(BOXES))
@pytest.mark.parametrize("charges", ["neutral", "plus3", "minus3", "zeros"])
def test_pme_oracle_against_direct_ewald(box_name, charges):
    box = BOXES[box_name]
    x, q = charged_system(box, 80, charges, seed=11)
    if charges == "zeros":
        assert (q == 0).sum() >= 15
    else:
        assert abs(q.sum() - {"neutral": 0, "plus3": 3, "minus3": -3}[charges]) < 1e-12
    errs = []
    for tol in (1e-3, 5e-4, 1e-5):
        for eps_r in (1.0, 4.0):
            ef, ee = _errors(x, q, box, 1.0, tol, eps_r)
            print(f"[{box_name} {charges} tol {tol:g} eps_r {eps_r:g}] K = {pme.pme_mesh_dims(box, pme.pme_alpha(1.0, tol), tol)} "
                  f"F {ef:.2e}  E {ee:.2e}")
            assert ef <= BARS[tol][0] and ee <= BARS[tol][1], (tol, eps_r, ef, ee)
        errs.append(ef)
    assert errs[0] > errs[1] > errs[2], errs  # the force error shrinks as error_tol does


def test_pme_oracle_mesh_shapes():
    """The systems above do reach the meshes the GPU matrix relies on: K = 6 (the minimum, both from the formula and
    from the clamp) and odd and even K."""
    ks = set()
    for box in BOXES.values():
        for tol in (1e-3, 5e-4, 1e-5):
            ks.update(pme.pme_mesh_dims(box, pme.pme_alpha(1.0, tol), tol))
    assert 6 in ks and any(k % 2 for k in ks) and any(k % 2 == 0 for k in ks)
    assert pme.pme_mesh_dims(np.array([0.5, 2.0, 2.0]), pme.pme_alpha(1.0, 1e-3), 1e-3)[0] == 6  # clamp of ceil(3.3)
