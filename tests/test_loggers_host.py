"""Host side of the device loggers (no GPU): the record schedule against Molly's rule, the gcd merge, the ctypes layout of
mb_log_t against the C header, and the refusal of loggers the engine does not record."""
import ctypes
import math
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

import mollyb200 as mb

capi = mb.capi
_LogPlan = sys.modules["molly_jl_b200"].api._LogPlan

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _molly_steps(n_steps, init_step, run_loggers, every):
    """simulate!(sys, ::VelocityVerlet, n_steps; init_step, run_loggers) with a GeneralObservableLogger(every): the steps
    apply_loggers! runs at (src/simulators.jl:575, :657; src/loggers.jl:44-56) filtered by s % every == 0 (:96-102)."""
    out = []
    if run_loggers is True and init_step % every == 0:  # apply_loggers!(..., init_step, ..., run_loggers == true)
        out.append(init_step)
    for s in range(init_step + 1, init_step + n_steps + 1):
        if (run_loggers is True or (run_loggers == "skipstart" and s != 0)) and s % every == 0:
            out.append(s)
    return out


@pytest.mark.parametrize("run_loggers", [True, False, "skipstart"])
def test_record_steps_follow_molly(run_loggers):
    for every in (1, 2, 3, 5, 7, 10, 100):
        for init_step in (0, 1, 3, 10, 99):
            for n_steps in (0, 1, 3, 12, 13, 100):
                assert mb.record_steps(every, n_steps, init_step, run_loggers) == _molly_steps(n_steps, init_step, run_loggers, every)


def test_run_loggers_is_checked():
    with pytest.raises(ValueError):
        mb.record_steps(5, 10, 0, "always")


class _Host:  # the attributes _LogPlan reads from a System with host state
    def __init__(self, loggers, n=4):
        self.loggers, self.n, self.k = loggers, n, mb.BOLTZMANN_K
        self.dtype = np.dtype(np.float32)
        self.coords = np.zeros((n, 3), np.float32)


@pytest.mark.parametrize("a,b", [(3, 5), (4, 6), (10, 10)])
def test_gcd_merge_and_each_logger_keeps_its_steps(a, b):
    """The engine records energies at gcd(a, b); each logger keeps exactly what Molly would log for it."""
    loggers = {"pe": mb.PotentialEnergyLogger(a), "ke": mb.KineticEnergyLogger(b), "x": mb.CoordinatesLogger(a),
               "v": mb.VelocitiesLogger(b)}
    host = _Host(loggers)
    n_steps, init_step = 37, 2
    plan = _LogPlan(host, n_steps, init_step, True)
    g = math.gcd(a, b)
    assert plan.desc.energy_every == g and plan.desc.coords_every == a and plan.desc.vels_every == b
    assert plan.steps["energy"] == _molly_steps(n_steps, init_step, True, g)
    assert plan.desc.energy_capacity == len(plan.steps["energy"]) and plan.desc.log_initial == 1
    # fake engine output: record k holds (step, pe = step, ke = 2 step); frames hold the step number
    e = plan.buf["energy"]
    e[:, 0] = plan.steps["energy"]
    e[:, 1] = e[:, 0]
    e[:, 2] = 2 * e[:, 0]
    for kind in ("coords", "vels"):
        for k, s in enumerate(plan.steps[kind]):
            plan.buf[kind][k] = s
    plan.push()
    assert [float(v) for v in loggers["pe"].history] == _molly_steps(n_steps, init_step, True, a)
    assert [float(v) / 2 for v in loggers["ke"].history] == _molly_steps(n_steps, init_step, True, b)
    assert [float(f[0, 0]) for f in loggers["x"].history] == _molly_steps(n_steps, init_step, True, a)
    assert [float(f[0, 0]) for f in loggers["v"].history] == _molly_steps(n_steps, init_step, True, b)


def test_derived_energy_loggers():
    loggers = {"t": mb.TemperatureLogger(1), "e": mb.TotalEnergyLogger(1)}
    host = _Host(loggers, n=10)
    plan = _LogPlan(host, 1, 0, "skipstart")
    assert plan.steps["energy"] == [1] and plan.desc.log_initial == 0
    plan.buf["energy"][0] = (1.0, -5.0, 3.0)
    plan.push()
    assert loggers["e"].history == [-2.0]
    assert loggers["t"].history[0] == pytest.approx(2 * 3.0 / (27 * mb.BOLTZMANN_K), rel=1e-15)
    assert mb.values(loggers["e"]) is loggers["e"].history


def test_unsupported_logger_raises_type_error():
    class ForcesLogger:
        n_steps = 10
    atoms = mb.atoms_from_arrays(np.ones(2), np.zeros(2), np.full(2, 0.3), np.full(2, 0.2), np.float32)
    with pytest.raises(TypeError, match="ForcesLogger"):
        mb.System(atoms=atoms, coords=np.zeros((2, 3)), boundary=mb.CubicBoundary(2.0), loggers={"f": ForcesLogger()})


@pytest.mark.skipif(shutil.which("gcc") is None, reason="needs a C compiler")
def test_mb_log_t_layout_matches_header(tmp_path):
    fields = [name for name, _ in capi.MBLog._fields_]
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "mollyb200.h"\nint main(void) {\n'
                   + "".join(f'    printf("%zu\\n", offsetof(mb_log_t, {f}));\n' for f in fields)
                   + '    printf("%zu\\n", sizeof(mb_log_t));\n    return 0;\n}\n')
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert got == [getattr(capi.MBLog, f).offset for f in fields] + [ctypes.sizeof(capi.MBLog)]


def test_simulate_vv_log_is_exported():
    assert "mb_simulate_vv_log" in capi.EXPORTED
    header = open(os.path.join(ROOT, "include", "mollyb200.h")).read()
    assert "int mb_simulate_vv_log(mb_ctx* ctx, void* coords, void* vels, const mb_vv_params_t* p, mb_log_t* log);" in header
