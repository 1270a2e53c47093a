"""Cost of Date32 columns on the device: table open with widened Date32 pages against the same values as an Int64 column
(the widening jobs FJ_DICT4 / FJ_WIDEN4 against FJ_DICT8 / FJ_COPY8), for dictionary and PLAIN pages, and a date-range
filter and GROUP BY d over a resident table.  Every answer is first checked against numpy.

    python tests/scripts/date32_probe.py [million rows, default 96] [repeats, default 5]

Writes its files to a temporary directory; prints one line per measurement, and the card's name and power limit."""
import datetime as dt
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from parseable_b200.query import DeviceTable, HostFile, StandardTableProvider, col, count_star  # noqa: E402

RG = 1 << 20


def write(path, days, dictionary):
    n = len(days)
    with pq.ParquetWriter(path, pa.schema([("d", pa.date32()), ("d64", pa.int64())]), use_dictionary=dictionary,
                          compression="none") as wr:
        for r0 in range(0, n, 8 * RG):
            part = days[r0:r0 + 8 * RG]
            wr.write_table(pa.table({"d": pa.array(part.astype(np.int32)).cast(pa.date32()), "d64": pa.array(part)}),
                           row_group_size=RG)


def timed(fn, repeats):
    fn()   # warm-up: module load, pools, pinned buffers
    ts = []
    for _ in range(repeats):
        t = time.perf_counter()
        out = fn()
        ts.append(1e3 * (time.perf_counter() - t))
        if isinstance(out, DeviceTable):
            out.close()
    return statistics.median(ts), min(ts), max(ts)


def main():
    n = int(sys.argv[1]) * 1_000_000 if len(sys.argv) > 1 else 96_000_000
    repeats = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(f"card: {card}; {n} rows, median / min / max of {repeats} runs", flush=True)
    rng = np.random.default_rng(1)
    days = rng.integers(18_000, 18_000 + 3650, n).astype(np.int64)   # ten years of dates
    with tempfile.TemporaryDirectory() as td:
        for form, dictionary in (("dictionary", True), ("PLAIN", False)):
            path = os.path.join(td, f"{form}.parquet")
            write(path, days, dictionary)
            hf = HostFile(path=path, pinned=True)
            for c in ("d", "d64"):
                med, lo, hi = timed(lambda: DeviceTable([hf], [c]), repeats)
                t = DeviceTable([hf], [c])
                print(f"open {form:10s} {c:4s}: {med:8.2f} ms ({lo:.2f} / {hi:.2f}), arena {t.device_bytes / 1e6:.0f} MB",
                      flush=True)
                t.close()
            if dictionary:
                lo_d, hi_d = 18_500, 19_500
                want = int(((days >= lo_d) & (days < hi_d)).sum())
                counts = np.bincount(days - 18_000)
                for c in ("d", "d64"):
                    t = DeviceTable([hf], [c])
                    prov = StandardTableProvider(t, schema={"d": pa.date32(), "d64": pa.int64()})
                    e0 = dt.date(1970, 1, 1)
                    lits = (e0 + dt.timedelta(days=lo_d), e0 + dt.timedelta(days=hi_d)) if c == "d" else (lo_d, hi_d)
                    flt = [(col(c) >= lits[0]) & (col(c) < lits[1])]
                    assert prov.scan(filters=flt, count_only=True).metrics["rows_selected"] == want
                    r = prov.aggregate([c], [count_star()]).table()
                    k = r[c].cast(pa.int32()).to_numpy() if c == "d" else r[c].to_numpy()
                    assert np.array_equal(r["count(*)"].to_numpy(), counts[k - 18_000]) and len(k) == np.count_nonzero(counts)
                    med, lo, hi = timed(lambda: prov.scan(filters=flt, count_only=True), repeats)
                    ks = prov.scan(filters=flt, count_only=True).metrics["scan_kernel_ms"]
                    print(f"filter {c:4s} range: {med:7.2f} ms per query ({lo:.2f} / {hi:.2f}), scan kernel {ks:.3f} ms", flush=True)
                    med, lo, hi = timed(lambda: prov.aggregate([c], [count_star()]), repeats)
                    ks = prov.aggregate([c], [count_star()]).metrics["scan_kernel_ms"]
                    print(f"GROUP BY {c:4s}: {med:7.2f} ms per query ({lo:.2f} / {hi:.2f}), scan kernel {ks:.3f} ms", flush=True)
                    t.close()
            hf.close()


if __name__ == "__main__":
    main()
