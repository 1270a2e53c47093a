"""Development probe (GPU box): the log search, SELECT * ... ORDER BY p_timestamp DESC LIMIT 100, under
PQ_QUERY_ALLGATHER with 2 and 4 ranks as processes on ONE device over the host-staged communicator build
(tools/libparseable_b200_hostcomm.so).  Not a bench line: bench.py is the contract.

    python tests/scripts/scan_merge_probe.py [row_groups=32] [steps=5] [ranks=2,4]

The synth logs (seeded, 262 144 rows per row group) sharded by row group.  Per rank and step (after one warm-up run) it
reports order_ms (the rank's own encode and sort), the merge kernels from the PQB_VERBOSE line (candidates: pack,
all-gather, row-id sort and scatter; the global sort; the projection by owner and the reductions of the result block)
and allreduce_ms, all CUDA-event times.  The all-gathers and all-reduces here are host-staged (files in an exchange
directory): their time says nothing about NCCL's."""
import json
import os
import re
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "scripts"))
from hashed_allreduce_probe import COLS, HOSTCOMM, ensure  # noqa: E402


def worker(rank, n, idfile, files, steps):
    import ctypes as C
    from ranks_worker import join
    from parseable_b200 import _lib as L
    from parseable_b200.query import DeviceTable, StandardTableProvider
    lib = L.load()
    assert lib.pq_init((C.c_int * 1)(0), 1) == 0, lib.pq_last_error(None)
    join(lib, L, idfile, n, rank)
    import pyarrow.parquet as pq
    schema = {f.name: f.type for f in pq.read_schema(files[0])}
    table = DeviceTable(files, COLS, shard_index=rank, shard_count=n)
    prov = StandardTableProvider(table, schema=schema)
    for step in range(steps + 1):   # step 0 warms up
        print(f"== step {step}", file=sys.stderr, flush=True)
        t0 = time.time()
        res = prov.scan(COLS, [], 100, row_ids=True, order_by=[("p_timestamp", "desc", False)], flags=L.PQ_QUERY_ALLGATHER)
        m = res.metrics
        print(json.dumps({"rank": rank, "step": step, "wall_s": time.time() - t0, "scan_kernel_ms": m["scan_kernel_ms"],
                          "order_ms": m["order_ms"], "allreduce_ms": m["allreduce_ms"], "rows_selected": m["rows_selected"]}), flush=True)
        sys.stderr.flush()
    table.close()
    lib.pq_comm_destroy()


def main():
    if len(sys.argv) > 1 and sys.argv[1] == "--rank":
        rank, n, idfile, steps = int(sys.argv[2]), int(sys.argv[3]), sys.argv[4], int(sys.argv[5])
        worker(rank, n, idfile, sys.argv[6:], steps)
        return
    nrg = int(sys.argv[1]) if len(sys.argv) > 1 else 32
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    ranks = [int(x) for x in (sys.argv[3] if len(sys.argv) > 3 else "2,4").split(",")]
    files = ensure(nrg)
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip(), f"| {nrg} row groups, {nrg * 262_144} rows", flush=True)
    merge_re = re.compile(r"scan merge: keep_r (\d+), keep_max (\d+), candidates (\d+), kept (\d+), sort path (\w+), exchange ([\d.]+) ms, "
                          r"candidates ([\d.]+) ms, sort ([\d.]+) ms, projection and reductions ([\d.]+) ms")
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
                for rec, mg in list(zip(recs, merges))[1:]:
                    kernels = float(mg[6]) + float(mg[7]) + float(mg[8])
                    print(f"n={n} rank {r} step {rec['step']}: scan {rec['scan_kernel_ms']:.2f} ms, order_ms {rec['order_ms']:.3f}, "
                          f"keep_r {mg[0]}, keep_max {mg[1]}, candidates {mg[2]}, path {mg[4]}, merge kernels {kernels:.3f} ms "
                          f"(candidates {float(mg[6]):.3f}, sort {float(mg[7]):.3f}, projection and reductions {float(mg[8]):.3f}; "
                          f"host-staged collectives included), exchange {float(mg[5]):.3f} ms, allreduce_ms {rec['allreduce_ms']:.3f}, "
                          f"rows_selected {rec['rows_selected']}, wall {rec['wall_s']:.2f} s", flush=True)
            for f in logs:
                f.close()


if __name__ == "__main__":
    main()
