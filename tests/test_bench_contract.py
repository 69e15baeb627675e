"""bench.py's reference arm (the UNMODIFIED reference from baseline/_ref on the host cores) under lookahead parallelism:
only rank 0 prints a result line.  Run on the tiny workload so that the CPU suite stays fast."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(extra_env=None, args=()):
    env = dict(os.environ)
    env.update(extra_env or {})
    return subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--workload", "tiny", *args],
                          capture_output=True, text=True, env=env, timeout=600, cwd=ROOT)


def test_reference_arm_other_ranks_exit_silently():
    res = _run(extra_env={"RANK": "1", "LOCAL_RANK": "1", "WORLD_SIZE": "2"})
    assert res.returncode == 0
    assert not [l for l in res.stdout.splitlines() if l.startswith("{")]
