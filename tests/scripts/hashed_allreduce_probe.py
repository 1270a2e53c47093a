"""Development probe (GPU box): a hashed GROUP BY under PQ_QUERY_ALLREDUCE, 2 and 4 ranks as processes on ONE device
over the host-staged communicator build (tools/libparseable_b200_hostcomm.so).  Not a bench line: bench.py is the
contract.

    python tests/scripts/hashed_allreduce_probe.py [row_groups=64] [steps=3] [ranks=2,4]

The synth logs (seeded, 262 144 rows per row group) grouped by host, pod, path with C4's aggregates: a key space far
wider than 2^26, so every rank fills a hashed table and the ranks merge them.  Per rank and step it reports the scan
kernel time, E_r (the groups it listed), G (the merged groups), and from the PQB_VERBOSE line the exchange, sort and fold
times (CUDA events).  The all-gathers here are host-staged (files in an exchange directory): their time is not NCCL's.
At the bench's full size (480 row groups) nearly every row is its own group, more than the 2^26 merged groups a query
may return, so the default is smaller."""
import json
import os
import re
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

COLS = ["p_timestamp", "host", "pod", "path", "status", "bytes", "latency_ms", "duration_s", "cpu"]
DIR = os.environ.get("PQB_PROBE_DIR", "/tmp/pqb_hashed_probe")
RGS_PER_FILE = 8
HOSTCOMM = os.path.join(ROOT, "tools", "libparseable_b200_hostcomm.so")


def _gen(args):
    path, first, n = args
    from parseable_b200 import synth
    if not os.path.exists(path):
        synth.write_logs16(path + ".tmp", n_row_groups=n, first_rg=first, columns=COLS)
        os.replace(path + ".tmp", path)
    return path


def ensure(nrg):
    import multiprocessing as mp
    os.makedirs(DIR, exist_ok=True)
    jobs = [(os.path.join(DIR, f"h_{g:05d}_{min(RGS_PER_FILE, nrg - g)}.parquet"), g, min(RGS_PER_FILE, nrg - g))
            for g in range(0, nrg, RGS_PER_FILE)]
    missing = [j for j in jobs if not os.path.exists(j[0])]
    if missing:
        with mp.get_context("spawn").Pool(max(1, min(len(missing), (os.cpu_count() or 2) - 1, 32))) as pool:
            pool.map(_gen, missing, chunksize=1)
    return [j[0] for j in jobs]


def worker(rank, n, idfile, files, steps):
    import ctypes as C
    sys.path.insert(0, os.path.join(ROOT, "tests", "scripts"))
    from ranks_worker import join
    from parseable_b200 import _lib as L
    from parseable_b200.query import DeviceTable, StandardTableProvider, count_star, max_, min_, sum_
    lib = L.load()
    assert lib.pq_init((C.c_int * 1)(0), 1) == 0, lib.pq_last_error(None)
    join(lib, L, idfile, n, rank)
    import pyarrow.parquet as pq
    schema = {f.name: f.type for f in pq.read_schema(files[0])}
    table = DeviceTable(files, COLS, shard_index=rank, shard_count=n)
    prov = StandardTableProvider(table, schema=schema)
    aggs = [count_star(), sum_("bytes"), min_("latency_ms"), max_("latency_ms"), sum_("duration_s"), max_("cpu")]
    for step in range(steps):
        print(f"== step {step}", file=sys.stderr, flush=True)
        t0 = time.time()
        res = prov.aggregate(["host", "pod", "path"], aggs, [], flags=L.PQ_QUERY_ALLREDUCE)
        m = res.metrics
        print(json.dumps({"rank": rank, "step": step, "wall_s": time.time() - t0, "scan_kernel_ms": m["scan_kernel_ms"],
                          "allreduce_ms": m["allreduce_ms"], "groups": m["groups_total"]}), flush=True)
        sys.stderr.flush()
    table.close()
    lib.pq_comm_destroy()


def main():
    if len(sys.argv) > 1 and sys.argv[1] == "--rank":
        rank, n, idfile, steps = int(sys.argv[2]), int(sys.argv[3]), sys.argv[4], int(sys.argv[5])
        worker(rank, n, idfile, sys.argv[6:], steps)
        return
    nrg = int(sys.argv[1]) if len(sys.argv) > 1 else 64
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    ranks = [int(x) for x in (sys.argv[3] if len(sys.argv) > 3 else "2,4").split(",")]
    files = ensure(nrg)
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip(), f"| {nrg} row groups, {nrg * 262_144} rows", flush=True)
    merge_re = re.compile(r"hashed merge: E_r (\d+), E_max (\d+), listed by all ranks (\d+), G (\d+), exchange ([\d.]+) ms, "
                          r"merge ([\d.]+) ms \(sort ([\d.]+) ms, fold ([\d.]+) ms\)")
    for n in ranks:
        with tempfile.TemporaryDirectory() as comm:
            env = {**os.environ, "PQB_LIB": HOSTCOMM, "PQB_COMM_DIR": comm, "PQB_VERBOSE": "1"}
            logs = [open(os.path.join(comm, f"log.{r}"), "w+") for r in range(n)]
            procs = [subprocess.Popen([sys.executable, os.path.abspath(__file__), "--rank", str(r), str(n), os.path.join(comm, "id"),
                                       str(steps)] + files, stdout=subprocess.PIPE, stderr=logs[r], text=True, env=env)
                     for r in range(n)]
            outs = [p.communicate()[0] for p in procs]
            for r, (p, o) in enumerate(zip(procs, outs)):
                logs[r].seek(0)
                merges = [m.groups() for m in merge_re.finditer(logs[r].read())]
                recs = [json.loads(x) for x in o.splitlines() if x.startswith("{")]
                if p.returncode:
                    print(f"n={n} rank {r}: exit {p.returncode}\n{o[-2000:]}")
                for rec, mg in zip(recs, merges):
                    print(f"n={n} rank {r} step {rec['step']}: scan {rec['scan_kernel_ms']:.2f} ms, E_r {mg[0]}, E_max {mg[1]}, "
                          f"listed {mg[2]}, G {mg[3]}, exchange {float(mg[4]):.2f} ms (host-staged), merge {float(mg[5]):.2f} ms "
                          f"(sort {float(mg[6]):.2f} ms, fold {float(mg[7]):.2f} ms), wall {rec['wall_s']:.2f} s", flush=True)
            for f in logs:
                f.close()


if __name__ == "__main__":
    main()
