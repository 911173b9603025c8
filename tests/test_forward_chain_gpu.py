"""The forward's launch chain (pytest -m gpu): programmatic dependent launch against fully serialised launches, bit for bit.

Every kernel of DeviceModel::forward is launched with programmatic dependent launch (PDL): it triggers its dependents at its start, so the
next grid becomes resident while its predecessor still runs, and several kernels do work before their griddepcontrol.wait — the stream-K
GEMM streams its first weight tiles (and L2 prefetches), decode attention streams the immutable K/V pages of its items, the stream-K
epilogue computes before it touches the shared workspace.  A kernel test launches one stage on inputs synced in beforehand, so none of this
overlap is exercised there.  OA_PDL=0 launches the same kernels with the same arguments, one after another.  The forward is deterministic bit
for bit (fixed stream-K / split-K summation orders, the attention merge in slot order), so the two must agree exactly: any difference in a
logit or an id is a read before the producer's write, or a write under a reader, somewhere in the chain.

Each case runs tests/chain_worker.py twice, as is and with OA_PDL=0 (the switch is read once per process).  The PDL worker runs its case
twice; both runs must equal each other and the serialised run, and a failure says which pair differs, so a run-to-run difference (a race
whose outcome varies, or nondeterminism) is told apart from a systematic one."""
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from chain_worker import CASES, STEPS  # noqa: E402


def _run_worker(case, out, repeat, pdl):
    """-> one dict of arrays per run"""
    env = dict(os.environ)
    env.pop("OA_PDL", None)
    if not pdl:
        env["OA_PDL"] = "0"
    r = subprocess.run([sys.executable, os.path.join(HERE, "chain_worker.py"), case, str(out), str(repeat)], env=env,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "CHAIN_OK" in r.stdout, f"{case} (PDL {'on' if pdl else 'off'}): rc={r.returncode}\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}"
    z = np.load(out)
    return [{key[len(f"r{k}_"):]: z[key] for key in z.files if key.startswith(f"r{k}_")} for k in range(repeat)]


def _mismatches(what, a, b):
    """-> one line per differing decode row / prefill row, with the largest logit difference where the full logits were kept"""
    msgs = []
    for step, row in zip(*np.nonzero((a["digests"] != b["digests"]) | (a["ids"] != b["ids"]))):
        full = {0: "first_step", STEPS - 1: "mixed_step"}.get(int(step))
        d = f"max|dlogit|={np.abs(a[full][row] - b[full][row]).max():.3e}" if full else "logits of this step not kept"
        msgs.append(f"{what}: decode step {step} row {row}: id {a['ids'][step, row]} vs {b['ids'][step, row]}, {d}")
    for row in np.nonzero(a["prefill_digests"] != b["prefill_digests"])[0]:
        msgs.append(f"{what}: prefill row {row}: arg-max {a['prefill_argmax'][row]} vs {b['prefill_argmax'][row]}, "
                    f"row max {a['prefill_max'][row]:.6f} vs {b['prefill_max'][row]:.6f}")
    return msgs


@pytest.mark.parametrize("case", list(CASES))
def test_dependent_launch_chain_is_bit_identical_to_serialised_launches(case, tmp_path):
    pdl = _run_worker(case, tmp_path / "pdl.npz", 2, True)
    serial, = _run_worker(case, tmp_path / "serial.npz", 1, False)
    _, batch, _ = CASES[case]
    assert pdl[0]["ids"].shape == (STEPS, batch) and pdl[0]["prefill_digests"].shape == (2048,)
    # two PDL runs that differ from each other: the chain is not reproducible (a race between overlapping kernels, or nondeterminism)
    again = _mismatches(f"{case} PDL run 1 vs run 2", pdl[0], pdl[1])
    msgs = again + _mismatches(f"{case} PDL run 1 vs serialised", pdl[0], serial) + _mismatches(f"{case} PDL run 2 vs serialised", pdl[1], serial)
    assert not msgs, (f"{len(msgs)} rows differ ({len(again)} between the two PDL runs):\n" + "\n".join(msgs[:20] + msgs[-20:]))
