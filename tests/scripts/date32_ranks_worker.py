"""One rank of Date32 queries across ranks on a single device (tests/test_date32_ranks.py): joins the communicator and
runs the cases below over its shard (row groups g % n == rank) of a resident table and of a file list, writing every
result as ranks_worker.py does (<out>/<case>.<source>.<rank>.arrow, or .json when refused).

Usage: date32_ranks_worker.py <rank> <nranks> <spec.json>; spec: {"files", "out", "idfile"}.  Meant for the host-staged
communicator build (PQB_LIB=tools/libparseable_b200_hostcomm.so, PQB_COMM_DIR)."""
import ctypes as C
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from ranks_worker import _write, join  # noqa: E402

from parseable_b200.query import QueryError, count, count_star, max_, min_  # noqa: E402

# name -> aggregate() arguments, run under PQ_QUERY_ALLREDUCE
AGGS = {
    "by_d": (["d"], [count_star(), count("d"), min_("d"), max_("d")]),
    "by_s": (["s"], [count_star(), count("d"), min_("d"), max_("d")]),
    "by_d_s": (["d", "s"], [count_star(), count("d")]),
    # (card(d) + 1) x (card(w) + 1) x (card(i) + 1) > 2^26: a hashed table on every rank, merged across them
    "hashed": (["d", "w", "i"], [count_star(), min_("d"), max_("d")]),
    "global": ([], [count_star(), count("d"), min_("d"), max_("d")]),
}
# name -> scan() arguments, run under PQ_QUERY_ALLGATHER
SCANS = {
    "order_asc": dict(projection=["d", "s"], row_ids=True, order_by=[("d", "asc")], limit=3000),
    "order_desc": dict(projection=["d"], row_ids=True, order_by=[("d", "desc")], limit=500),
}


def main():
    rank, n = int(sys.argv[1]), int(sys.argv[2])
    spec = json.load(open(sys.argv[3]))
    import pyarrow.parquet as pq
    from parseable_b200 import _lib as L
    from parseable_b200.query import DeviceTable, StandardTableProvider
    lib = L.load()
    dev = (C.c_int * 1)(int(os.environ.get("PQB_RANK_DEVICE", "0")))
    assert lib.pq_init(dev, 1) == 0, lib.pq_last_error(None)
    join(lib, L, spec["idfile"], n, rank)
    files, out = spec["files"], spec["out"]
    schema = {}
    for p in files:
        for fld in pq.read_schema(p):
            schema.setdefault(fld.name, fld.type)
    table = DeviceTable(files, list(schema), shard_index=rank, shard_count=n)
    provs = {"table": StandardTableProvider(table, schema=schema),
             "files": StandardTableProvider(files, schema=schema, shard_index=rank, shard_count=n)}
    for src, prov in provs.items():
        for name, (keys, aggs) in AGGS.items():
            path = os.path.join(out, f"{name}.{src}.{rank}")
            try:
                _write(path, None, res=prov.aggregate(keys, aggs, flags=L.PQ_QUERY_ALLREDUCE))
            except QueryError as e:
                _write(path, None, err=e)
        for name, kw in SCANS.items():
            path = os.path.join(out, f"{name}.{src}.{rank}")
            try:
                _write(path, None, res=prov.scan(flags=L.PQ_QUERY_ALLGATHER, **kw))
            except QueryError as e:
                _write(path, None, err=e)
    table.close()
    assert lib.pq_comm_destroy() == 0
    print(f"rank {rank}/{n}: done", flush=True)


if __name__ == "__main__":
    main()
