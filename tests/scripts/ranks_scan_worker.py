"""One rank of ORDER BY ... LIMIT scans under PQ_QUERY_ALLGATHER on a single device (tests/test_ranks_scan_order.py):
joins the communicator, runs the case list below over its shard (row groups g % n == rank) of a resident table and of
a file list, and writes every result as ranks_worker.py does (<out>/<case>.<source>.<rank>.arrow, or .json when
refused), with <...>.meta.json holding rows_selected.  Rank 0 also runs every case without the flag over all files
(<out>/<case>.ref.0.arrow): the answer of one rank over the unsharded table.

Before each query it writes "== <case>.<source>" to stderr, so that with PQB_VERBOSE the test can tell which query
printed which line.  Usage: ranks_scan_worker.py <rank> <nranks> <spec.json>; spec: {"files", "out", "idfile"}."""
import ctypes as C
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from ranks_worker import _write, filters_of, join  # noqa: E402

from parseable_b200.query import QueryError, Window, count_star  # noqa: E402

ALL = ["ts", "s", "sp", "i", "f", "b", "x", "w", "opt"]   # every column kind: Timestamp (DELTA), Utf8 (dictionary / PLAIN), Int64, Float64, Boolean
# name -> scan() arguments; every one runs under PQ_QUERY_ALLGATHER on both sources
CASES = {
    "log_search": dict(projection=ALL, row_ids=True, order_by=[("ts", "desc", False)], limit=100, batch_size=32),
    "ties_b": dict(projection=["b", "rid"], row_ids=True, order_by=[("b", "asc")], limit=5000),   # cut inside the FALSE tie
    "s_nulls_first": dict(projection=["s", "rid"], order_by=[("s", "asc", True)], limit=50_000),   # past the all-NULL row group
    "s_nulls_last": dict(projection=["s"], row_ids=True, order_by=[("s", "desc", False)], limit=400),
    "opt_nulls_first": dict(projection=["opt", "rid"], order_by=[("opt", "asc", True)], limit=100_000),   # absent from one file
    # (`rid` too: a file-list rank whose files hold none of the columns it reads has no flat store, and refuses an ordered scan)
    "opt_nulls_last": dict(projection=["opt", "rid"], row_ids=True, order_by=[("opt", "desc", False)], limit=30_000),
    "f_total": dict(projection=["f"], row_ids=True, order_by=[("f", "asc")], limit=2000),
    "f_total_desc": dict(projection=["f", "s"], row_ids=True, order_by=[("f", "desc", False)], limit=3000),
    "s_dict": dict(projection=["s", "i"], row_ids=True, order_by=[("s", "asc")], limit=1000),
    "sp_plain": dict(projection=["sp"], row_ids=True, order_by=[("sp", "desc", False)], limit=700),   # the PLAIN row group's values
    "sp_ties": dict(projection=["sp", "x"], row_ids=True, order_by=[("sp", "asc", False)], limit=5000),
    "three_terms": dict(projection=["b", "s", "f", "sp"], row_ids=True, order_by=[("b", "desc", False), ("s", "asc", False), ("f", "desc", False)],
                        limit=2500),
    "row_ids_only": dict(order_by=[("x", "asc")], limit=500),
    "some_empty": dict(projection=["ts", "s"], row_ids=True, order_by=[("ts", "desc", False)], limit=200, filters=[("ts_lt", 3)]),
    "all_empty": dict(projection=["ts", "s"], row_ids=True, order_by=[("ts", "desc", False)], limit=200, filters=[("i_eq", -999_999)]),
    "limit_0": dict(projection=["x", "s"], row_ids=True, order_by=[("x", "desc", False)], limit=0),
    "limit_past": dict(projection=["x", "s"], row_ids=True, order_by=[("x", "desc", False)], limit=1_000_000, filters=[("x_gt", 490)]),
    "json": dict(projection=["ts", "s", "f", "b", "opt"], order_by=[("ts", "desc", False)], limit=100, json="lines"),
    # Utf8 terms of a column absent from the second file, and of one in no file (every rank joins the agreement)
    "sopt": dict(projection=["sopt", "rid"], row_ids=True, order_by=[("sopt", "asc", False)], limit=3000),
    "ghost": dict(projection=["ghost", "s"], row_ids=True, order_by=[("ghost", "asc"), ("s", "desc", False)], limit=300),
    # only `opt`: at n = 8 a file-list rank holding second-file row groups only reads no page at all, has no flat store
    # and refuses an ordered scan, so every rank refuses (REFUSED_AT)
    "opt_only": dict(projection=["opt"], row_ids=True, order_by=[("opt", "desc", False)], limit=1000),
}
REFUSED_AT = {"opt_only": (8, "files")}   # (n, source) where every rank refuses the case
AGAIN = ["s_dict", "sp_ties"]   # run again on the resident table (the agreed Utf8 numbering is kept), and after rank 1 reopens it
# test switches set on one rank only: its merge budget is too small / its items all take the path without flat-store
# copies, which an ordered scan refuses before the scan.  Every rank must refuse.
REFUSALS = {"refuse_budget": ("PQB_MERGE_BUDGET", "4096"), "refuse_flat": ("PQB_FLAT_SCAN", "0")}


def victim(n):
    return min(1, n - 1)


def scan(prov, case, flags):
    kw = dict(case)
    flt = filters_of(kw.pop("filters", []))
    return prov.scan(filters=flt, flags=flags, **kw)


def run(prov, case, out, flags):
    t0 = time.time()
    try:
        res = scan(prov, case, flags)
    except QueryError as e:
        _write(out, None, err=e, seconds=time.time() - t0)
        return
    _write(out, None, res=res)
    with open(out + ".meta.json", "w") as f:
        json.dump({"rows_selected": res.metrics["rows_selected"], "allreduce_ms": res.metrics["allreduce_ms"],
                   "order_ms": res.metrics["order_ms"]}, f)


def misuse(prov, L, out, rank, with_comm=True):
    """The flag where it does not apply: {name: [code, message]}."""
    AG = L.PQ_QUERY_ALLGATHER
    got = {}
    tries = {
        "aggregate": lambda: prov.aggregate(["b"], [count_star()], flags=AG),
        "count_only": lambda: prov.scan(count_only=True, flags=AG),
        "window": lambda: prov.scan(["s"], order_by=[("x", "asc")], window=Window(partition_by=["b"], fetch=2), flags=AG),
        "no_order_by": lambda: prov.scan(["s"], limit=10, flags=AG),
    }
    if not with_comm:
        tries = {"no_comm": lambda: prov.scan(["s"], order_by=[("x", "asc")], limit=10, flags=AG)}
    for name, fn in tries.items():
        try:
            fn()
            got[name] = None
        except QueryError as e:
            got[name] = [e.code, e.message]
    with open(os.path.join(out, f"misuse{'' if with_comm else '_nocomm'}.{rank}.json"), "w") as f:
        json.dump(got, f)


def main():
    rank, n = int(sys.argv[1]), int(sys.argv[2])
    spec = json.load(open(sys.argv[3]))
    import pyarrow as pa
    import pyarrow.parquet as pq
    from parseable_b200 import _lib as L
    from parseable_b200.query import DeviceTable, StandardTableProvider
    lib = L.load()
    dev = (C.c_int * 1)(int(os.environ.get("PQB_RANK_DEVICE", "0")))
    assert lib.pq_init(dev, 1) == 0, lib.pq_last_error(None)
    files, out = spec["files"], spec["out"]
    schema = {}
    for p in files:
        for fld in pq.read_schema(p):
            schema.setdefault(fld.name, fld.type)
    schema["ghost"] = pa.string()   # a Utf8 column in no file: NULL in every row
    cols = list(schema)
    whole = StandardTableProvider(files, schema=schema)
    if rank == 0:
        misuse(whole, L, out, rank, with_comm=False)
        for name, case in CASES.items():   # the unsharded answer, without the flag
            _write(os.path.join(out, f"{name}.ref.0"), None, res=scan(whole, case, 0))
    join(lib, L, spec["idfile"], n, rank)
    AG = L.PQ_QUERY_ALLGATHER

    def go(prov, name, case, src):
        print(f"== {name}.{src}", file=sys.stderr, flush=True)
        run(prov, case, os.path.join(out, f"{name}.{src}.{rank}"), AG)
        sys.stderr.flush()

    table = DeviceTable(files, cols, shard_index=rank, shard_count=n)
    provs = {"table": StandardTableProvider(table, schema=schema),
             "files": StandardTableProvider(files, schema=schema, shard_index=rank, shard_count=n)}
    for src, prov in provs.items():
        for name, case in CASES.items():
            go(prov, name, case, src)
        for name in REFUSALS if n > 1 else []:
            var, value = REFUSALS[name]
            if rank == victim(n):
                os.environ[var] = value
            try:
                go(prov, name, CASES["log_search"], src)
            finally:
                os.environ.pop(var, None)
            go(prov, "after_" + name, CASES["log_search"], src)
    misuse(provs["table"], L, out, rank)
    if n > 1:
        # __row_id is global only over one file list that every rank shards by row group: an unsharded provider, and
        # rank 0 opening a shorter list, are refused by every rank
        go(whole, "refuse_unsharded", CASES["log_search"], "files")
        go(StandardTableProvider(files if rank else files[:1], schema=schema, shard_index=rank, shard_count=n), "refuse_lists",
           CASES["log_search"], "files")
        go(provs["files"], "after_refuse_lists", CASES["log_search"], "files")
    # the agreed Utf8 numbering kept with the resident table: the same queries again, then after rank 1 alone reopens
    # its table (every rank then agrees anew)
    prov = provs["table"]
    for step in ("again", "reopen"):
        if step == "reopen" and rank == 1:
            table.close()
            table = DeviceTable(files, cols, shard_index=rank, shard_count=n)
            prov = StandardTableProvider(table, schema=schema)
        for name in AGAIN:
            go(prov, f"{step}_{name}", CASES[name], "table")
    table.close()
    assert lib.pq_comm_destroy() == 0
    print(f"rank {rank}/{n}: done", flush=True)


if __name__ == "__main__":
    main()
