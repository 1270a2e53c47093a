"""Multi-GPU ORDER BY check: one process per GPU, row groups sharded g % n == rank, partial tables merged by the NCCL
all-reduce (PQ_QUERY_ALLREDUCE), then ordered and cut on every rank.  Every rank must hold the oracle's whole-table
GROUP BY sorted the same way on the host, and print the same digest of its rows as every other rank.  The orders are
total (every GROUP BY key is a term), so the expected rows do not depend on slot order.
Usage: mgpu_order_check.py <rank> <nranks> <idfile> <files...>"""
import ctypes as C
import hashlib
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))   # tests/scripts/ -> repo root
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    rank, n, idfile = int(sys.argv[1]), int(sys.argv[2]), sys.argv[3]
    files = sys.argv[4:]
    import pyarrow as pa
    from parseable_b200 import _lib as L
    from parseable_b200.query import StandardTableProvider, col, count_star, max_, sum_
    from test_order_by import canon, host_order
    lib = L.load()
    dev = (C.c_int * 1)(int(os.environ.get("PQB_RANK_DEVICE", rank)))   # PQB_RANK_DEVICE: every rank on one device
    assert lib.pq_init(dev, 1) == 0, lib.pq_last_error(None)
    if rank == 0:
        buf = C.create_string_buffer(L.PQ_COMM_ID_BYTES)
        assert lib.pq_comm_unique_id(buf) == 0
        with open(idfile + ".tmp", "wb") as f:
            f.write(buf.raw)
        os.replace(idfile + ".tmp", idfile)
        ident = buf.raw
    else:
        t0 = time.time()
        while not os.path.exists(idfile):
            if time.time() - t0 > 120:
                raise SystemExit("timeout waiting for the NCCL id")
            time.sleep(0.05)
        ident = open(idfile, "rb").read()
    assert lib.pq_comm_init_rank(ident, n, rank) == 0, lib.pq_last_error(None)

    from oracle.oracle import Oracle
    ora = Oracle.from_parquet(files)
    schema = {f.name: f.type for f in ora.table.schema}
    prov = StandardTableProvider(files, schema=schema, shard_index=rank, shard_count=n)
    cs = count_star()
    cases = [
        # a Utf8 key (ranks over the agreed numbering) and an aggregate term, cut
        ("host_by_count", ["host"], [cs, sum_("bytes")], [(cs, "desc"), ("host", "asc")], 25, []),
        # an Int64 key read from the agreed dictionary, DESC, with a Utf8 key after it, cut
        ("status_host", ["host", "status"], [cs, max_("latency_ms")], [("status", "desc"), ("host", "asc")], 40, []),
        # a full order (no cut) with a filter
        ("level_full", ["level"], [cs], [(cs, "asc"), ("level", "desc")], None, [col("latency_ms") > 50]),
    ]
    for name, keys, aggs, order, limit, flt in cases:
        got = prov.aggregate(keys, aggs, flt, flags=L.PQ_QUERY_ALLREDUCE, order_by=order, limit=limit)
        t = got.table()
        exp = ora.group_by(keys, aggs, flt)
        terms = [(a.name if hasattr(a, "fn") else a, d == "desc", d == "desc") for a, d in order]
        idx = host_order(exp, terms)
        exp = exp.take(pa.array(idx[:limit] if limit is not None else idx, pa.int64()))
        assert got.metrics["groups"] == exp.num_rows, (rank, name, got.metrics["groups"], exp.num_rows)
        assert canon(t) == canon(exp.select(t.column_names)), (rank, name)
        digest = hashlib.sha256(repr(canon(t)).encode()).hexdigest()
        print(f"rank {rank}: ordered digest {name} {digest}", flush=True)
    print(f"rank {rank}/{n}: multi-GPU ORDER BY parity OK", flush=True)
    lib.pq_comm_destroy()


if __name__ == "__main__":
    main()
