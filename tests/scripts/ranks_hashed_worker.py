"""One rank of a multi-rank hashed GROUP BY on a single device (tests/test_ranks_hashed.py): joins the communicator, runs
the case list below under PQ_QUERY_ALLREDUCE over its shard (row groups g % n == rank) of a resident table and of a file
list, and writes every result as ranks_worker.py does (<out>/<case>.<source>.<rank>.arrow, or .json when refused).

Before each query it writes "== <case>.<source>" to stderr, so that with PQB_VERBOSE the test can tell which query
printed which plan line.  Usage: ranks_hashed_worker.py <rank> <nranks> <spec.json>; spec: {"files", "out", "idfile"}."""
import ctypes as C
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from ranks_worker import FP, _write, join, run_case  # noqa: E402,F401

from parseable_b200.query import Window, avg, count, count_star, date_bin, max_, min_, sum_  # noqa: E402

MINUTE = 60_000
# every key tuple below is wider than 2^26 combinations in the ranks' agreed numbering; ("u", "i") is narrower on every
# rank alone (test_ranks_hashed.py sizes the values so)
CASES = {
    "fp_u_i": (["u", "i"], FP, [], {}),
    "fp_u_f": (["u", "f"], FP, [], {}),
    "fp_u_b_bin": (["u", "b", date_bin(MINUTE, "ts")], FP, [], {}),
    "fp_u_opt_i": (["u", "opt", "i"], FP, [], {}),     # `opt` is absent from the second file
    "agg_x_w": (["u", "i"], [count("x"), sum_("x"), avg("x"), min_("x"), max_("x"), sum_("w")], [], {}),
    "agg_fn": (["u", "f"], [count("fn"), sum_("fn"), avg("fn"), min_("fn"), max_("fn"), min_("rid"), max_("rid")], [], {}),
    "minmax_str_bool": (["u", "i"], [min_("sp"), max_("sp"), min_("b"), max_("b"), count("b")], [], {}),
    "where": (["u", "i"], FP, [("x_gt", 0)], {}),
    "nothing": (["u", "i"], FP, [("x_gt", 1_000_000)], {}),
    "pruned": (["u", "b", date_bin(MINUTE, "ts")], FP, [("ts_lt", 3)], {}),   # every row group of some ranks pruned
    "order_limit": (["u", "i"], [count_star(), sum_("x")], [],
                    {"order_by": [(count_star(), "desc"), ("u", "asc"), ("i", "asc")], "limit": 7}),
    "order_ties": (["u", "i"], [count_star(), sum_("x")], [], {"order_by": [(count_star(), "desc")], "limit": 25}),
    "window": (["b", "u", "i"], [count_star(), sum_("rid")], [],
               {"order_by": [(count_star(), "desc"), ("u", "asc"), ("i", "asc")],
                "window": Window(partition_by=["b"], fetch=3, row_number=True)}),
    "json": (["u", "i"], [count_star(), sum_("x"), max_("sp")], [], {"json": "lines"}),
}
AGAIN = ["fp_u_i", "order_ties"]     # run a second time: the same rows in the same order
LOCAL = ["fp_u_i"]                   # without PQ_QUERY_ALLREDUCE: dense on every rank alone
# test switches set on one rank only: its table runs full / its merge budget is too small.  Every rank must refuse.
REFUSALS = {"refuse_full": ("PQB_HASH_SLOTS", "1024"), "refuse_budget": ("PQB_MERGE_BUDGET", "4096")}


def victim(n):
    return min(1, n - 1)


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
    AR = L.PQ_QUERY_ALLREDUCE

    def go(prov, name, case, src, flags=AR):
        print(f"== {name}.{src}", file=sys.stderr, flush=True)
        run_case(prov, case, os.path.join(out, f"{name}.{src}.{rank}"), flags)
        sys.stderr.flush()

    table = DeviceTable(files, list(schema), shard_index=rank, shard_count=n)
    provs = {"table": StandardTableProvider(table, schema=schema),
             "files": StandardTableProvider(files, schema=schema, shard_index=rank, shard_count=n)}
    for src, prov in provs.items():
        for name, case in CASES.items():
            go(prov, name, case, src)
        for name in AGAIN:
            go(prov, "again_" + name, CASES[name], src)
        for name in LOCAL:
            go(prov, "local_" + name, CASES[name], src, flags=0)
        for name, (var, value) in REFUSALS.items():
            if rank == victim(n):
                os.environ[var] = value
            try:
                go(prov, name, CASES["fp_u_i"], src)
            finally:
                os.environ.pop(var, None)
            go(prov, "after_" + name, CASES["fp_u_i"], src)
    table.close()
    assert lib.pq_comm_destroy() == 0
    print(f"rank {rank}/{n}: done", flush=True)


if __name__ == "__main__":
    main()
