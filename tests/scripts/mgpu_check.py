"""Multi-GPU parity check: one process per GPU, row groups sharded g % n == rank, partial
aggregate tables merged by ONE NCCL all-reduce inside libparseable_b200.so; every rank must
hold the oracle's answer for the WHOLE table.  Usage: mgpu_check.py <rank> <nranks> <idfile> <files...>"""
import ctypes as C
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))   # tests/scripts/ -> repo root
sys.path.insert(0, ROOT)


def main():
    rank, n, idfile = int(sys.argv[1]), int(sys.argv[2]), sys.argv[3]
    files = sys.argv[4:]
    split = []          # after "--": one file per rank, only some of them with NULLs (the ranks' footers disagree about NULL presence)
    if "--" in files:
        i = files.index("--")
        files, split = files[:i], files[i + 1:]
    from parseable_b200 import _lib as L
    from parseable_b200.query import StandardTableProvider, col, count_star, sum_, min_, max_, avg, count
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
    import math
    ora = Oracle.from_parquet(files)
    schema = {f.name: f.type for f in ora.table.schema}
    prov = StandardTableProvider(files, schema=schema, shard_index=rank, shard_count=n)
    cases = [
        (["host", "status"], [count_star(), sum_("bytes"), min_("latency_ms"), max_("latency_ms"), sum_("duration_s"), max_("cpu")], []),
        (["level"], [count_star(), avg("latency_ms"), count("cpu")], [col("status") == 200]),
        ([], [count_star(), sum_("bytes"), min_("cpu")], [col("level") == "ERROR"]),
        ([], [count_star()], [(col("level") == "ERROR") & (col("latency_ms") > 100)]),
        (["region"], [count_star()], [col("level") == "NOPE"]),
        # a key column without a dictionary (PLAIN doubles): the rows are interned per rank, the numbering agreed across ranks
        (["status", "cpu"], [count_star(), max_("bytes")], [col("latency_ms") > 150]),
    ]
    for keys, aggs, flt in cases:
        print(f"rank {rank}: case {keys} {len(aggs)} aggs", flush=True)
        got = prov.aggregate(keys, aggs, flt, flags=L.PQ_QUERY_ALLREDUCE)
        exp = ora.group_by(keys, aggs, flt)
        res = got.table() if got.batches else exp.slice(0, 0)
        if keys:
            order = [(k, "ascending") for k in keys]
            res, exp = res.sort_by(order), exp.sort_by(order)
        assert res.num_rows == exp.num_rows, (rank, keys, res.num_rows, exp.num_rows)
        for name in exp.column_names:
            a, b = res[name].to_pylist(), exp[name].to_pylist()
            if a != b:
                ok = len(a) == len(b) and all((x is None and y is None) or (x is not None and y is not None and
                                              math.isclose(x, y, rel_tol=1e-9)) for x, y in zip(a, b))
                assert ok and (name.startswith("sum(") or name.startswith("avg(")), (rank, keys, name)
    if split:
        # one rank's shard is NULL-free, the other's is not: COUNT(col) / AVG / SUM must still be the whole table's
        # (the null_count == 0 shortcut is a per-rank footer decision and is off under PQ_QUERY_ALLREDUCE)
        ora2 = Oracle.from_parquet(split)
        prov2 = StandardTableProvider(split, schema={f.name: f.type for f in ora2.table.schema}, shard_index=rank, shard_count=n)
        for keys, aggs, flt in [(["level"], [count_star(), count("cpu"), avg("cpu"), sum_("bytes"), min_("latency_ms")], []),
                                ([], [count("host"), count("bytes"), max_("cpu")], [col("status") == 200])]:
            got = prov2.aggregate(keys, aggs, flt, flags=L.PQ_QUERY_ALLREDUCE).table()
            exp = ora2.group_by(keys, aggs, flt)
            if keys:
                order = [(k, "ascending") for k in keys]
                got, exp = got.sort_by(order), exp.sort_by(order)
            for name in exp.column_names:
                a, b = got[name].to_pylist(), exp[name].to_pylist()
                ok = a == b or all((x is None and y is None) or (x is not None and y is not None and math.isclose(x, y, rel_tol=1e-9)) for x, y in zip(a, b))
                assert ok, (rank, "split", keys, name, a[:5], b[:5])
        print(f"rank {rank}: ranks that disagree about NULL presence still agree on the answer", flush=True)
    print(f"rank {rank}/{n}: multi-GPU all-reduce parity OK", flush=True)
    lib.pq_comm_destroy()


if __name__ == "__main__":
    main()
