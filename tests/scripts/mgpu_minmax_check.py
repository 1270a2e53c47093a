"""MIN / MAX over Utf8 / Boolean under PQ_QUERY_ALLREDUCE: one process per GPU, row groups sharded g % n == rank, the
partial MIN / MAX cells (ranks in the numbering every rank agreed on) merged by the library's NCCL all-reduce; every rank
must hold the CPU restatement's answer for the WHOLE table.  Usage: mgpu_minmax_check.py <rank> <nranks> <idfile> <files...>"""
import ctypes as C
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))   # tests/scripts/ -> repo root
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    rank, n, idfile = int(sys.argv[1]), int(sys.argv[2]), sys.argv[3]
    files = sys.argv[4:]
    from parseable_b200 import _lib as L
    from parseable_b200.query import StandardTableProvider, col, count_star, date_bin, max_, min_, sum_
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
    try:
        from oracle.oracle import Oracle
        from test_min_max_strings import assert_matches, expect
        ora = Oracle.from_parquet(files)
        schema = {f.name: f.type for f in ora.table.schema}
        prov = StandardTableProvider(files, schema=schema, shard_index=rank, shard_count=n)
        cases = [
            ([], [min_("host"), max_("host"), max_("path"), count_star()], []),
            (["status"], [min_("pod"), max_("pod"), sum_("bytes")], []),
            (["host"], [min_("host"), max_("level")], [col("latency_ms") > 500]),   # the key column is also the input
            ([date_bin("1m")], [min_("service"), max_("message")], []),
            (["region"], [min_("path")], [col("level") == "NOPE"]),
            ([], [min_("level"), max_("level")], [col("level") == "NOPE"]),
        ]
        for keys, aggs, flt in cases:
            print(f"rank {rank}: case {keys} {[a.name for a in aggs]}", flush=True)
            for _ in range(2):   # the second run reads the agreement kept with the table column
                got = prov.aggregate(keys, aggs, flt, flags=L.PQ_QUERY_ALLREDUCE)
                exp = expect(ora, keys, aggs, flt)
                if got.batches:
                    assert_matches(got.table(), exp, keys, aggs)
                else:   # a grouped query over zero rows: no groups, no batches
                    assert keys and exp == {}, exp
        print(f"rank {rank}: parity OK", flush=True)
    finally:
        lib.pq_comm_destroy()


if __name__ == "__main__":
    main()
