"""bench.py contract pieces that run without a GPU: the reference arm (`--impl reference`: the CPU port of the reference algorithm
on the host cores, one JSON line with the contract keys) and the workload labels and algorithmic bytes the report uses."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_prints_one_json_line_with_the_contract_keys():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--workload", "C2", "--steps", "2", "--warmup", "3"],
                       capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["metric"] == "checkresources_decisions_per_sec" and d["unit"] == "decisions/s"
    assert d["higher_is_better"] is True and d["value"] > 0 and d["steps"] == 2 and d["warmup"] == 3 and d["n_gpus"] == 1
    assert d["cpu_baseline"]["kind"] in ("port", "reference") and d["cpu_baseline"]["cores"] >= 1 and d["cpu_baseline"]["value"] == d["value"]
    assert d["e2e"] == {"value": d["value"], "unit": "decisions/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert d["config"]["workload"].startswith("C2:")


def test_reference_arm_does_no_work_on_other_ranks():
    env = dict(os.environ, RANK="1", WORLD_SIZE="2")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2"], capture_output=True, text=True, timeout=120, cwd=ROOT, env=env)
    assert r.returncode == 0 and r.stdout.strip() == ""


def test_workload_labels_and_algorithmic_bytes():
    sys.path.insert(0, ROOT)
    import bench
    import workloads as W
    assert bench.workload_label(W.C3(), 1, 1 << 24).startswith("C3:")
    assert bench.workload_label(W.C3(), 8, 1 << 24).startswith("C4: the C3 table, 8 x 2^24 requests")
    for name, per_request in (("C2", 73), ("C3", 197), ("C5", 489)):   # the roofline's bytes per request (SURVEY.md 8(d))
        assert W.WORKLOADS[name]().bytes_per_request() == per_request, name
