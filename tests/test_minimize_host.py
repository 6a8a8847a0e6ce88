"""CPU tests of the steepest-descent minimiser: the numpy restatement (tests/sd_oracle.py) against the reference's own
minimisation test (test/minimization.jl), and the Python-level argument checks of SteepestDescentMinimizer / simulate."""
import io

import numpy as np
import pytest

import mollyb200 as mb
import sd_oracle as sdo

X0 = np.array([[1.0, 1.0, 1.0], [1.6, 1.0, 1.0], [1.4, 1.6, 1.0]])
SIGMA = np.full(3, 0.4 / 2 ** (1 / 6))
EPS = np.ones(3)
BOX = np.full(3, 5.0)


def _dists(x):
    out = []
    for i, j in ((0, 1), (0, 2), (1, 2)):
        d = x[j] - x[i]
        d -= BOX * np.round(d / BOX)
        out.append(np.linalg.norm(d))
    return np.array(out)


def test_oracle_reproduces_reference_minimization():
    """test/minimization.jl: 3 LJ atoms, tol 1 -> all distances 0.4 nm +- 1e-3, PE -3.0 +- 1e-4 (the CPU tolerances)."""
    x, trace = sdo.steepest_descent(X0, BOX, lambda x: sdo.lj_energy_forces(x, BOX, SIGMA, EPS), step_size=0.01, tol=1.0)
    assert np.all(np.abs(_dists(x) - 0.4) < 1e-3)
    _, e = sdo.lj_energy_forces(x, BOX, SIGMA, EPS)
    assert abs(e - (-3.0)) < 1e-4
    # the trace: record 0 is the start, accepted energies decrease, the last iteration's max force is below tol
    assert trace[0, 0] == 0 and trace[0, 3] == 1 and np.isnan(trace[0, 2])
    acc = trace[trace[:, 3] == 1, 1]
    assert np.all(np.diff(acc) < 0)
    assert trace[-1, 2] < 1.0 and np.all(trace[1:-1, 2] >= 1.0)
    assert len(trace) < 1001


def test_oracle_zero_forces_rejects_once():
    """Two atoms beyond any interaction (zero forces): x + h F / 0 is NaN, the trial is rejected and the loop stops (m < tol)."""
    zero = lambda x: (np.zeros_like(x), 0.0)  # noqa: E731
    x, trace = sdo.steepest_descent(np.array([[0.5, 0.5, 0.5], [3.0, 3.0, 3.0]]), BOX, zero, tol=1.0)
    assert len(trace) == 2 and trace[1, 3] == 0 and np.isnan(trace[1, 1]) and trace[1, 2] == 0
    assert np.array_equal(x, [[0.5, 0.5, 0.5], [3.0, 3.0, 3.0]])


def test_minimizer_arguments():
    assert mb.SteepestDescentMinimizer() == mb.SteepestDescentMinimizer(step_size=0.01, max_steps=1000, tol=1000.0)
    for bad in (dict(step_size=0.0), dict(step_size=-1.0), dict(max_steps=-1), dict(tol=-1.0), dict(step_size=float("nan"))):
        with pytest.raises(ValueError):
            mb.SteepestDescentMinimizer(**bad)


def _system():
    atoms = mb.atoms_from_arrays(np.ones(3), np.zeros(3), SIGMA, EPS, np.float64)
    return mb.System(atoms=atoms, coords=X0, boundary=mb.CubicBoundary(5.0), pairwise_inters=(mb.LennardJones(),),
                     dtype=np.float64)


def test_simulate_dispatch_checks_before_any_engine_call():
    """These are refused before the engine is touched (they hold without a GPU)."""
    s = _system()
    with pytest.raises(NotImplementedError):
        mb.simulate(s, mb.SteepestDescentMinimizer(), run_loggers=True)
    with pytest.raises(NotImplementedError):
        mb.simulate(s, mb.SteepestDescentMinimizer(), run_loggers="skipstart")
    with pytest.raises(TypeError):
        mb.simulate(s, mb.SteepestDescentMinimizer(), 10)
    with pytest.raises(TypeError):
        mb.simulate(s, mb.VelocityVerlet(dt=0.002))  # VelocityVerlet still needs n_steps
    with pytest.raises(TypeError):
        mb.simulate(s, object(), 10)
    with pytest.raises(ValueError):
        mb.simulate(s, mb.VelocityVerlet(dt=0.002), 10, run_loggers="sometimes")
    assert s._ctx is None


def test_log_lines_follow_the_reference_format():
    trace = np.array([[0, -1.5, np.nan, 1], [1, -2.25, 3.5, 1], [2, np.nan, 0.0, 0]])
    assert mb.sd_log_lines(trace) == ["Step 0 - potential energy -1.5 - max force N/A - N/A",
                                      "Step 1 - potential energy -2.25 - max force 3.5 - accepted",
                                      "Step 2 - potential energy nan - max force 0.0 - rejected"]
    buf = io.StringIO()
    for line in mb.sd_log_lines(trace[:1]):
        print(line, file=buf)
    assert buf.getvalue() == "Step 0 - potential energy -1.5 - max force N/A - N/A\n"
