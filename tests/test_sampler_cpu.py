"""The CPU sampler's token and log-prob streams, pinned exactly: unseeded rows draw from the engine's seeded CPU
generator, so any change to how the sampler keys or shapes its random draws shows up here (`mp_sampler_streams.py`
has the request mix). One process and TP2 over gloo (the vocab-parallel sampler), with async scheduling on and off.

Re-record after an intended change of the streams: `python tests/test_sampler_cpu.py`."""
from conftest import scratch_dir
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "sampler_cpu_streams.json")
CASES = [(1, False, 0), (1, True, 0), (2, False, 29741), (2, True, 29751)]


def _key(tp, async_on):
    return f"tp{tp}_{'async' if async_on else 'sync'}"


def _run(tp, async_on, port, out_dir):
    out = os.path.join(out_dir, f"{_key(tp, async_on)}.json")
    env = dict(os.environ, PYTHONPATH=ROOT, GLLM_B200_LOG="WARNING", GLLM_TEST_ASYNC="1" if async_on else "0",
               OMP_NUM_THREADS="1")
    script = os.path.join(ROOT, "tests", "mp_sampler_streams.py")
    if tp == 1:
        cmd = [sys.executable, script, "1", out]
    else:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={tp}",
               "--master-addr", "127.0.0.1", "--master-port", str(port), script, str(tp), out]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, env=env, cwd=ROOT)
    assert r.returncode == 0 and os.path.exists(out), r.stdout[-2000:] + r.stderr[-3000:]
    with open(out) as f:
        return json.load(f)


@pytest.mark.parametrize("tp,async_on,port", CASES)
def test_cpu_sampler_streams_match_the_golden_file(tp, async_on, port):
    with open(GOLDEN) as f:
        want = json.load(f)[_key(tp, async_on)]
    got = _run(tp, async_on, port, scratch_dir("gllm_b200_streams_"))
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        assert g[0] == w[0], (i, "tokens")
        assert g[1] == w[1], (i, "logprobs")


if __name__ == "__main__":
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        rec = {_key(tp, a): _run(tp, a, port, d) for tp, a, port in CASES}
    with open(GOLDEN, "w") as f:
        json.dump(rec, f)
