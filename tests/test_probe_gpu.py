"""Engine configurations checked in their own process (tests/probe_worker.py): GQA group 8 — what one rank of Llama-3-70B TP=8 runs —
and group 1, an engine whose text goes through a trained byte-level BPE tokenizer, and the scheduler's mixed steps (decoding sequences
ride along in prefill steps: both attention kernels in one forward, staggered arrivals as the reference's one-goroutine-per-request
callers produce them — pkg/handlers/execute.go:205)."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.mark.parametrize("probe", ["tiny-llama-g8", "tiny-llama-mha", "bpe", "mixed"])
def test_probe(probe):
    r = subprocess.run([sys.executable, os.path.join(HERE, "probe_worker.py"), probe], capture_output=True, text=True, timeout=240)
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-2000:])
