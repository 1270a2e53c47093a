"""Development probe (GPU box): regular-expression filters against their LIKE equivalents, table resident.

Each query's count is first checked against the RE2 / C oracle (test_regex.RxOracle) on one whole file.  Then, alternated,
scan_kernel_ms and device_ms of:
  * message ~ 'timeout-xy+zzy'  vs  message LIKE '%timeout-xyzzy%'   (dictionary message: both read a per-entry LUT)
  * the same two on files rewritten with `message` undictionaried (PLAIN pages: the per-row DFA walk), also as string
    bytes walked per second
  * level = 'ERROR' AND message ~ '...'
  * a (?i) alternation
Prints the card's name and power limit.  Not a bench line: bench.py is the contract.

    python tests/scripts/regex_probe.py [row_groups=96] [plain_files=2] [steps=20]   (8 row groups per file)
"""
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    import numpy as np
    import pyarrow.compute as pc
    import pyarrow.parquet as pq
    from parseable_b200.query import DeviceTable, StandardTableProvider, col
    from test_regex import RxOracle
    nrg = int(sys.argv[1]) if len(sys.argv) > 1 else 96
    nplain = int(sys.argv[2]) if len(sys.argv) > 2 else 2
    steps = int(sys.argv[3]) if len(sys.argv) > 3 else 20
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"card: {card}", flush=True)
    from parseable_b200 import synth
    cols = ["message", "level", "latency_ms"]
    td_data = tempfile.mkdtemp(prefix="rx_probe_")   # the bench files carry no `message`: logs16 row groups with it
    files = []
    for i in range(0, nrg, 8):
        f = os.path.join(td_data, f"logs16_{i:04d}.parquet")
        synth.write_logs16(f, n_row_groups=min(8, nrg - i), first_rg=i, columns=["p_timestamp"] + cols)
        files.append(f)
    Q = {
        "regex token": [col("message").regex("timeout-xy+zzy")],
        "like token": [col("message").like("%timeout-xyzzy%")],
        "level AND regex": [(col("level") == "ERROR") & col("message").regex(r"upstream (cache|db) (miss|hit)")],
        "(?i) alternation": [col("message").regex(r"(?i)PANIC|expired token|RESET PEER")],
    }
    ora = RxOracle.from_parquet(files[0], columns=cols)
    schema = {f.name: f.type for f in pq.read_schema(files[0])}
    p1 = StandardTableProvider([files[0]], schema=schema)
    for name, flt in Q.items():
        got = p1.scan(filters=flt, count_only=True).metrics["rows_selected"]
        assert got == ora.count(flt), (name, got, ora.count(flt))
    print(f"parity ok on {files[0]} ({ora.n} rows)", flush=True)

    def run(prov, name, flt, nbytes=None):
        for _ in range(3):
            prov.scan(filters=flt, count_only=True)
        scan, dev = [], []
        for _ in range(steps):
            r = prov.scan(filters=flt, count_only=True)
            scan.append(r.metrics["scan_kernel_ms"])
            dev.append(r.metrics["device_ms"])
        med = lambda v: sorted(v)[len(v) // 2]
        extra = f" | {nbytes / (med(scan) * 1e-3) / 1e9:.2f} GB/s of string bytes walked" if nbytes else ""
        print(f"{name:28s} scan_kernel_ms p50 {med(scan):8.3f} (min {min(scan):.3f}, max {max(scan):.3f}) | device_ms p50 "
              f"{med(dev):8.3f} | rows {r.metrics['rows_selected']}{extra}", flush=True)

    table = DeviceTable(files, cols)
    prov = StandardTableProvider(table, schema=schema)
    print(f"dictionary message: {table.rows} rows in {nrg} row groups", flush=True)
    for _ in range(2):
        for name, flt in Q.items():
            run(prov, name, flt)
    table.close()

    with tempfile.TemporaryDirectory() as td:
        plain, nbytes = [], 0
        for i, f in enumerate(files[:nplain]):
            t = pq.read_table(f, columns=cols)
            p = os.path.join(td, f"plain_{i}.parquet")
            pq.write_table(t, p, compression="NONE", use_dictionary=["level"], row_group_size=1 << 18)
            nbytes += int(pc.sum(pc.binary_length(t["message"].cast("string"))).as_py() or 0)
            plain.append(p)
        ora = RxOracle.from_parquet(plain[0])
        pp = StandardTableProvider([plain[0]], schema=schema)
        for name in ("regex token", "like token"):
            assert pp.scan(filters=Q[name], count_only=True).metrics["rows_selected"] == ora.count(Q[name]), name
        table = DeviceTable(plain, cols)
        prov = StandardTableProvider(table, schema=schema)
        print(f"PLAIN message: {table.rows} rows in {len(plain)} files, {nbytes / 1e9:.2f} GB of message bytes", flush=True)
        for _ in range(2):
            run(prov, "regex token (PLAIN)", Q["regex token"], nbytes)
            run(prov, "like token (PLAIN)", Q["like token"], nbytes)
        run(prov, "(?i) alternation (PLAIN)", Q["(?i) alternation"], nbytes)
        table.close()
    import shutil
    shutil.rmtree(td_data, ignore_errors=True)


if __name__ == "__main__":
    main()
