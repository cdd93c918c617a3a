"""bench.py host-side contract (no GPU): the CPU arm sizes itself to the cores the container really
has, non-zero ranks exit quietly, and our arm refuses to run without CUDA."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(extra_env=None, *args):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    env.update(extra_env or {})
    return subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), *args], env=env,
                          capture_output=True, text=True, timeout=600)


def test_host_cores_respects_affinity():
    sys.path.insert(0, ROOT)
    import bench
    n = bench.host_cores()
    assert 1 <= n <= (os.cpu_count() or 1)
    if hasattr(os, "sched_getaffinity"):
        assert n <= len(os.sched_getaffinity(0))


def test_reference_arm_other_ranks_are_silent():
    r = _run({"RANK": "1", "WORLD_SIZE": "2"}, "--impl", "reference", "--gpus", "2", "--steps", "1",
             "--warmup", "0")
    assert r.returncode == 0 and r.stdout.strip() == ""


def test_our_arm_refuses_to_run_without_cuda():
    r = _run(None, "--steps", "1", "--warmup", "0", "--no-cpu-baseline")
    assert r.returncode != 0 and "CUDA" in (r.stderr + r.stdout)


def test_dump_outputs_only_where_implemented():
    r = _run(None, "--workload", "rvae", "--steps", "1", "--warmup", "0", "--dump-outputs",
             os.path.join(ROOT, "never_written"))
    assert r.returncode != 0 and "--dump-outputs" in r.stderr
    assert not os.path.exists(os.path.join(ROOT, "never_written"))
