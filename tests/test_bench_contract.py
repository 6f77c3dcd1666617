"""bench.py contract checks that need no GPU: the reference (CPU) arm prints ONE JSON line with the keys the driver
reads, ranks other than 0 stay silent, and the GPU arm's line (a committed run) carries the required objects."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REQUIRED = {"metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
            "vs_baseline", "dtype", "data", "config", "e2e", "cpu_baseline"}


def _run(env_extra, *args):
    env = dict(os.environ, **env_extra)
    return subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), *args], env=env, capture_output=True,
                          text=True, timeout=600)


def test_reference_arm_prints_one_json_line():
    r = _run({}, "--impl", "reference", "--steps", "1", "--warmup", "1", "--cpu-chunks", "1")
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [ln for ln in r.stdout.splitlines() if ln.strip()]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert REQUIRED <= set(d) and d["impl"] == "reference" and d["metric"] == "kv_encode_decode_raw_GBps"
    assert d["value"] > 0 and d["e2e"]["value"] == d["value"] and d["e2e"]["h2d_bytes_per_step"] == 0
    assert d["cpu_baseline"]["kind"] == "port" and "workload" in d["config"]
    # the arm must use the host's threads (round 2 once pinned itself onto one core before counting them): every visible
    # one, or -- where a cgroup grants fewer CPUs than it shows -- whichever of {visible, granted, 2 x granted} ran fastest
    sys.path.insert(0, ROOT)
    import bench
    ncpu, quota = len(os.sched_getaffinity(0)), bench._cgroup_cpus()
    allowed = {ncpu} | ({min(ncpu, quota), min(ncpu, 2 * quota)} if quota else set())
    assert d["cpu_baseline"]["cores"] in allowed and d["cpu_baseline"]["cores"] >= min(allowed)


def test_reference_arm_other_ranks_are_silent():
    r = _run({"RANK": "1", "WORLD_SIZE": "2", "LOCAL_RANK": "1"}, "--impl", "reference", "--gpus", "2")
    assert r.returncode == 0 and r.stdout.strip() == ""


def test_committed_gpu_line_has_the_contract_objects():
    d = json.loads(open(os.path.join(ROOT, "profiles", "h100_bench.json")).read().strip().splitlines()[-1])
    assert REQUIRED <= set(d) and {"roofline", "clocks", "gpu_launches"} <= set(d)
    rl = d["roofline"]
    assert {"bound", "achieved", "peak", "unit", "frac", "traffic"} <= set(rl) and rl["bound"] == "hbm"
    assert abs(rl["frac"] - rl["achieved"] / rl["peak"]) < 1e-3
    assert d["e2e"]["h2d_bytes_per_step"] > 0 and d["e2e"]["d2h_bytes_per_step"] > 0 and d["gpu_launches"] > 0
    assert d["cpu_baseline"]["kind"] in ("port", "reference")
    # round 2: the end-to-end number goes through the engine, the sweep carries parity checks, the container is version 3
    assert "LMCacheEngine.store" in d["e2e"]["path"] and d["e2e"]["value"] > 0
    sweep = d["config"]["entropy_sweep"]
    assert len(sweep) == 5 and all(x["parity_spot_check"] == "bit-exact" for x in sweep)
    assert max(x["coder_bits_per_symbol"] for x in sweep) > 3.5 and "v3" in d["config"]["coder"]
