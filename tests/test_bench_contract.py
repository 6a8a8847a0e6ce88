"""bench.py contract pieces: the reference arm (CPU restatement timed on the host cores) and, on a GPU, --dump-outputs."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_prints_one_json_line():
    # C3 (6mrr) is the workload the oracle finishes in seconds; the driver calls the same entry with its own K / W
    p = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--workload", "c3",
                        "--gpus", "1", "--steps", "1000", "--warmup", "100"], capture_output=True, text=True, timeout=600,
                       cwd=ROOT)
    assert p.returncode == 0, p.stderr[-2000:]
    lines = [l for l in p.stdout.strip().splitlines() if l.startswith("{")]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["metric"] == "md_steps_per_sec" and d["unit"] == "steps/s"
    assert d["higher_is_better"] is True and d["n_gpus"] == 1 and d["value"] > 0
    # a bounded sample of whole neighbour-list periods, however many steps were asked for
    assert d["steps"] % 10 == 0 and d["steps"] <= 60
    assert d["e2e"] == {"value": d["value"], "unit": d["unit"], "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    cb = d["cpu_baseline"]
    assert cb["kind"] == "port" and cb["cores"] >= 1 and cb["value"] == d["value"] and "sample" in cb


@pytest.mark.gpu
def test_dump_outputs_are_reproducible(tmp_path):
    # two runs with the same arguments time exactly --steps steps and dump the same arrays, bit for bit
    dumps = []
    for k in range(2):
        out = tmp_path / f"run{k}"
        p = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--workload", "c2", "--gpus", "1", "--steps", "20",
                            "--warmup", "5", "--no-cpu-baseline", "--no-e2e", "--dump-outputs", str(out)],
                           capture_output=True, text=True, timeout=600, cwd=ROOT)
        assert p.returncode == 0, p.stderr[-2000:]
        d = json.loads([l for l in p.stdout.strip().splitlines() if l.startswith("{")][-1])
        assert d["steps"] == 20
        arrs = {name: np.load(out / f"{name}.npy") for name in ("coords", "velocities")}
        for a in arrs.values():
            assert a.dtype == np.float32 and a.shape == (d["config"]["n_atoms"], 3) and np.isfinite(a).all()
        dumps.append(arrs)
    for name in dumps[0]:
        assert np.array_equal(dumps[0][name], dumps[1][name]), name


def test_reference_arm_other_ranks_exit_quietly():
    env = dict(os.environ, RANK="1", WORLD_SIZE="2", LOCAL_RANK="1")
    p = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2"],
                       capture_output=True, text=True, timeout=120, cwd=ROOT, env=env)
    assert p.returncode == 0 and p.stdout.strip() == ""
