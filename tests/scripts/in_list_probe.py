"""Development probe (GPU box): IN lists against the OR chains and the single EQ leaf they replace, table resident.

  * logs16 `host` (dictionary pages): host = 'x', host IN (k hosts) for k = 1, 16, 10 000, and the 16-leaf OR chain;
  * a PLAIN-page Utf8 column of 16-hex-digit trace ids (no dictionary: the per-row set probe), IN (k ids) for k = 1,
    1 000 and 10^6, half of them present.
Each count is checked against pyarrow first.  Prints, per query, the median scan_kernel_ms (CUDA events around the scan
kernel) and device_ms of `steps` COUNT_ONLY scans, and the card's name and power limit.  Not a bench line: bench.py is.

    python tests/scripts/in_list_probe.py [row_groups=48] [steps=20]   (8 row groups per file)
"""
import os
import subprocess
import sys
import tempfile
from functools import reduce

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)


def main():
    import numpy as np
    import pyarrow as pa
    import pyarrow.compute as pc
    import pyarrow.parquet as pq
    from parseable_b200 import synth
    from parseable_b200.query import DeviceTable, StandardTableProvider, col
    nrg = int(sys.argv[1]) if len(sys.argv) > 1 else 48
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 20
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"card: {card}", flush=True)
    td = tempfile.mkdtemp(prefix="in_probe_")
    files = []
    for i in range(0, nrg, 8):
        f = os.path.join(td, f"logs16_{i:04d}.parquet")
        synth.write_logs16(f, n_row_groups=8, first_rg=i, columns=["host", "level"])
        files.append(f)
    host = pa.concat_tables([pq.read_table(f, columns=["host"]) for f in files])["host"].cast(pa.string())
    hosts = pc.unique(host).to_pylist()
    rng = np.random.default_rng(1)
    # the trace-id files: one PLAIN Utf8 column, the same row count
    tfiles, tids = [], []
    for k, f in enumerate(files):
        n = pq.ParquetFile(f).metadata.num_rows
        ids = np.array([f"{int(v):016x}" for v in rng.integers(0, 1 << 62, n)], dtype=object)
        tids.append(ids)
        p = os.path.join(td, f"trace_{k:04d}.parquet")
        pq.write_table(pa.table({"trace_id": pa.array(ids, pa.string())}), p, use_dictionary=False, compression="NONE",
                       row_group_size=synth.ROW_GROUP)
        tfiles.append(p)
    trace = pa.array(np.concatenate(tids), pa.string())
    print(f"{len(host)} rows, {len(hosts)} distinct hosts", flush=True)

    def run(prov, flt, want, label):
        got = prov.scan(filters=flt, count_only=True).metrics["rows_selected"]
        assert got == want, (label, got, want)
        ks, ds = [], []
        for _ in range(steps):
            m = prov.scan(filters=flt, count_only=True).metrics
            ks.append(m["scan_kernel_ms"])
            ds.append(m["device_ms"])
        print(f"{label:44s} selected {want:>10d}  scan_kernel_ms {np.median(ks):7.3f}  device_ms {np.median(ds):7.3f}", flush=True)

    dt = DeviceTable(files, ["host", "level"])
    try:
        prov = StandardTableProvider(dt)
        one = hosts[0]
        run(prov, [col("host") == one], int(pc.sum(pc.equal(host, one)).as_py() or 0), "host = 'x'")
        for k in (1, 16, 10_000):
            vals = [hosts[int(i)] for i in rng.integers(0, len(hosts), min(k, len(hosts)))]
            vals += [f"absent-{i}" for i in range(k - len(vals))]
            want = int(pc.sum(pc.is_in(host, value_set=pa.array(vals, pa.string()))).as_py() or 0)
            run(prov, [col("host").isin(vals)], want, f"host IN ({k})")
            if k == 16:
                run(prov, [reduce(lambda a, b: a | b, [col("host") == v for v in vals])], want, "16-leaf OR chain of host = 'x'")
    finally:
        dt.close()
    dt = DeviceTable(tfiles, ["trace_id"])
    try:
        prov = StandardTableProvider(dt)
        present = trace.to_pylist()
        for k in (1, 1000, 1_000_000):
            vals = [present[int(i)] for i in rng.integers(0, len(present), k - k // 2)] + [f"{int(v):016x}x" for v in range(k // 2)]
            want = int(pc.sum(pc.is_in(trace, value_set=pa.array(vals, pa.string()))).as_py() or 0)
            run(prov, [col("trace_id").isin(vals)], want, f"trace_id IN ({k}), PLAIN pages")
    finally:
        dt.close()


if __name__ == "__main__":
    main()
