"""bench.py's reference arm (`--impl reference`) runs on the host cores only, so its contract is checkable without a GPU: one
JSON line with the native arm's metric / unit / workload string, `impl`, `cpu_baseline` (kind, cores, sample) and the e2e
object; under torchrun every rank but 0 exits 0 without work.  (The native arm needs an H100: `pytest -m gpu`.)"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(extra_env, *flags):
    env = dict(os.environ, **extra_env)
    return subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", *flags], cwd=ROOT, env=env,
                          capture_output=True, text=True, timeout=900)


def test_reference_arm_prints_the_contract_line():
    sys.path.insert(0, ROOT)
    import bench
    r = _run({}, "--gpus", "1", "--steps", "1", "--warmup", "0")
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.splitlines() if l.strip()]
    assert len(lines) == 1                                            # ONE JSON line on stdout, nothing else
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["metric"] == bench.METRIC and d["unit"] == "steps/s" and d["higher_is_better"] is True
    assert d["steps"] == 1 and d["warmup"] == 0 and d["n_gpus"] == 1 and d["data"] == "synthetic" and d["dtype"] == "f32"
    assert d["config"]["workload"] == bench.WORKLOAD                  # the native arm's workload, verbatim
    assert abs(d["value"] - 1e3 / d["ms_per_step"]) < 1e-9 * d["value"] + 1e-12
    cb = d["cpu_baseline"]
    assert cb["kind"] in ("reference", "port") and cb["cores"] >= 1 and cb["value"] == d["value"] and "512 rays" in cb["sample"]
    assert d["e2e"] == {"value": d["value"], "unit": "steps/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    from oracle import make_ref
    assert cb["kind"] == ("reference" if make_ref.available() else "port")


def test_reference_arm_other_ranks_exit_without_work():
    r = _run({"RANK": "1", "LOCAL_RANK": "1", "WORLD_SIZE": "2"}, "--gpus", "2", "--steps", "1", "--warmup", "0")
    assert r.returncode == 0 and r.stdout.strip() == "", (r.stdout[-500:], r.stderr[-500:])
