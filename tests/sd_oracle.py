"""numpy restatement of simulate!(sys, ::SteepestDescentMinimizer) (src/simulators.jl:183-274), TEST INFRASTRUCTURE.

The loop runs over a force-and-energy function of the caller's choice (the C oracle's all-pairs or neighbour-list loops,
oracle/bonded.py, oracle/pme.py), so the arithmetic is independent of the engine's. Forces at the restored coordinates of
a rejected trial are the forces computed there before the trial: the reference recomputes them and gets the same values.
Returns the final coordinates and the same records as mb_minimize_sd: (step, E or E_trial, max force, accepted)."""
import numpy as np


def wrap(x, box):
    return x - np.floor(x / box) * box  # wrap_coords, src/spatial.jl:573-579


def steepest_descent(x, box, fe, step_size=0.01, max_steps=1000, tol=1000.0, init_step=0, wrap_fn=None):
    """fe(x) -> (forces (n,3), energy). Float64 throughout. wrap_fn(x): wrap_coords of another boundary (default: the
    rectangular box `box`)."""
    box = np.asarray(box, np.float64)
    wrap_fn = wrap_fn or (lambda y: wrap(y, box))
    x = wrap_fn(np.asarray(x, np.float64))
    F, E = fe(x)
    trace = [(init_step, E, np.nan, 1.0)]
    h = step_size
    for step_n in range(init_step + 1, init_step + max_steps + 1):
        m = np.sqrt(np.max(np.einsum("ij,ij->i", F, F)))
        x_copy = x
        with np.errstate(divide="ignore", invalid="ignore"):
            x = wrap_fn(x + h * F / m)
        if np.all(np.isfinite(x)):
            F_trial, E_trial = fe(x)
        else:
            F_trial, E_trial = F, np.nan
        if E_trial < E:
            h = 6 * h / 5
            E = E_trial
            F = F_trial
            trace.append((step_n, E_trial, m, 1.0))
        else:
            x = x_copy
            h = h / 5
            trace.append((step_n, E_trial, m, 0.0))
        if m < tol:
            break
    return x, np.array(trace, np.float64)


def lj_energy_forces(x, box, sigma, eps):
    """Plain LennardJones (NoCutoff, minimum image) for a handful of atoms: src/interactions/lennard_jones.jl:79-140."""
    n = len(x)
    f = np.zeros_like(x)
    e = 0.0
    for i in range(n):
        for j in range(i + 1, n):
            dr = x[j] - x[i]
            dr -= box * np.round(dr / box)
            r2 = dr @ dr
            s2 = (0.5 * (sigma[i] + sigma[j])) ** 2 / r2
            ep = np.sqrt(eps[i] * eps[j])
            s6 = s2 ** 3
            e += 4 * ep * (s6 * s6 - s6)
            fv = (24 * ep * (2 * s6 * s6 - s6) / r2) * dr
            f[i] -= fv
            f[j] += fv
    return f, e
