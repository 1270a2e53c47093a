import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def built():
    """The in-tree shared libraries; build them when missing (nvcc cross-compiles without a GPU)."""
    import subprocess
    if not (os.path.exists(os.path.join(ROOT, "parseable_b200", "libparseable_b200.so"))
            and os.path.exists(os.path.join(ROOT, "tools", "libdecode_core_host.so"))
            and os.path.exists(os.path.join(ROOT, "oracle", "liboracle.so"))):
        subprocess.check_call(["make", "-C", ROOT, "-j4", "all"])
    return ROOT


@pytest.fixture(scope="session")
def data_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("pqb"))


@pytest.fixture(scope="session")
def small_files(data_dir):
    """Two small logs16 files (no nulls / 2 % nulls), 3 row groups of 70 000 rows: several pages per
    column chunk, dictionary growth inside a chunk, PLAIN fallback for the all-distinct f64 columns."""
    from parseable_b200 import synth
    out = {}
    for tag, rate in (("nn", 0.0), ("nulls", 0.02)):
        p = os.path.join(data_dir, f"small_{tag}.parquet")
        synth.write_logs16(p, n_row_groups=3, rows_per_group=70_000, null_rate=rate)
        out[tag] = p
    return out
