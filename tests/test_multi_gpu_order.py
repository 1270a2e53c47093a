"""ORDER BY ... LIMIT under PQ_QUERY_ALLREDUCE on real GPUs: one process per GPU; every rank returns the oracle's
ordered, cut result for the whole table, and the same rows as every other rank."""
import os
import re
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _device_count():
    from parseable_b200 import _lib as L
    return L.load().pq_device_count()


def test_two_rank_ordered_allreduce(small_files, tmp_path, built):
    if _device_count() < 2:
        pytest.skip("needs 2 GPUs")
    n = 2
    idfile = str(tmp_path / "nccl_id")
    procs = [subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", "scripts", "mgpu_order_check.py"), str(r), str(n), idfile,
                               small_files["nulls"], small_files["nn"]], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
             for r in range(n)]
    outs = [p.communicate(timeout=600)[0] for p in procs]
    digests = []
    for r, (p, o) in enumerate(zip(procs, outs)):
        assert p.returncode == 0, f"rank {r}:\n{o[-3000:]}"
        assert "ORDER BY parity OK" in o
        digests.append(dict(re.findall(r"ordered digest (\S+) (\S+)", o)))
    assert len(digests[0]) == 3 and all(d == digests[0] for d in digests), digests
