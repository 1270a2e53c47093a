"""One rank of a multi-rank run on a single device (tests/test_ranks_one_gpu.py): joins the communicator, runs the case
list below over its shard (row groups g % n == rank, g global across the files) of a resident table and of a file
list, and writes every result to <out>/<case>.<source>.<rank>.arrow (Arrow IPC), or <...>.json ({code, message,
seconds}) when the query is refused.

Usage: ranks_worker.py <rank> <nranks> <spec.json>; spec: {"files", "nostats", "out", "idfile"}.  Meant for the
host-staged communicator build (PQB_LIB=tools/libparseable_b200_hostcomm.so, PQB_COMM_DIR); PQB_RANK_DEVICE picks
the device (default 0)."""
import ctypes as C
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))   # tests/scripts/ -> repo root
sys.path.insert(0, ROOT)

from parseable_b200.query import (Window, avg, col, count, count_distinct, count_star, date_bin, max_, median,  # noqa: E402
                                  min_, sum_)

HOUR = 3_600_000
FP = [count_star(), count("rid"), sum_("rid"), min_("rid"), max_("rid"), sum_("rnd")]
# the row groups' ts ranges are disjoint and ascending (test_ranks_one_gpu.py): this bound keeps row groups 0-2 only
TS_CUT = ("ts_lt", 3)

# name -> (keys, aggs, filters, extra aggregate() arguments); every one runs under PQ_QUERY_ALLREDUCE on both sources
CASES = {
    "fp_s": (["s"], FP, [], {}),
    "fp_sp": (["sp"], FP, [], {}),
    "fp_i": (["i"], FP, [], {}),
    "fp_f": (["f"], FP, [], {}),
    "fp_b": (["b"], FP, [], {}),
    "fp_opt": (["opt"], FP, [], {}),                       # absent from the second file: NULL on some ranks only
    "fp_s_b": (["s", "b"], FP, [], {}),
    "fp_i_f_b": (["i", "f", "b"], FP, [], {}),
    "fp_sp_b_opt": (["sp", "b", "opt"], FP, [], {}),
    "fp_bin": ([date_bin(HOUR, "ts")], FP, [], {}),
    "fp_bin_s": ([date_bin(7 * HOUR, "ts", 1234), "s"], FP, [], {}),
    "fp_bin_pruned": ([date_bin(HOUR, "ts")], FP, [TS_CUT], {}),   # every row group of some ranks pruned
    "fp_s_where": (["s"], FP, [("x_gt", 0)], {}),
    "agg_x": (["b"], [count("x"), sum_("x"), avg("x"), min_("x"), max_("x")], [], {}),
    "agg_w": (["s"], [count("w"), sum_("w"), min_("w"), max_("w")], [], {}),
    "agg_f": (["b"], [count("f"), sum_("f"), avg("f"), min_("f"), max_("f")], [], {}),
    # without NaN and +-inf every SUM / AVG of `f` is exact too: the cross-rank Float64 sum itself, not only NaN-ness
    "agg_f_finite": (["b"], [count("f"), sum_("f"), avg("f"), min_("f"), max_("f")], [("f_gt", -1000), ("f_lt", 1000)], {}),
    "agg_f_by_i": (["i"], [min_("f"), max_("f"), sum_("x"), count("x")], [], {}),
    "minmax_str": (["b"], [min_("s"), max_("s"), min_("sp"), max_("sp")], [], {}),
    "minmax_str_by_s": (["s"], [min_("sp"), max_("sp"), count("sp")], [], {}),
    "minmax_bool": (["s"], [min_("b"), max_("b"), count("b")], [], {}),
    "global": ([], [count_star(), count("x"), sum_("x"), sum_("w"), min_("w"), max_("w"), min_("s"), max_("sp")], [], {}),
    "global_where": ([], [count_star(), sum_("rid"), min_("f"), max_("b")], [("x_gt", 0)], {}),
    "count_only": ([], [count_star()], [("x_gt", 0)], {}),
    "nothing": (["s"], FP, [("i_eq", -999_999)], {}),
    "nothing_global": ([], [count_star(), sum_("x"), min_("s")], [("i_eq", -999_999)], {}),
    "order_limit": (["s"], [count_star(), sum_("x")], [], {"order_by": [(count_star(), "desc"), ("s", "asc")], "limit": 7}),
    "window": (["b", "s"], [count_star(), sum_("rid")], [],
               {"order_by": [(count_star(), "desc"), ("s", "asc")], "window": Window(partition_by=["b"], fetch=3, row_number=True)}),
    "json": (["b", "s"], [count_star(), sum_("x"), max_("sp")], [], {"json": "lines"}),
}
# run without PQ_QUERY_ALLREDUCE: each rank's answer over its own shard
LOCAL = ["fp_s", "fp_sp", "fp_f", "agg_x", "minmax_str", "fp_bin"]
# under PQ_QUERY_ALLREDUCE every rank refuses these: COUNT(DISTINCT) / MEDIAN for every rank alike, the others because
# of what one rank's shard holds (PLAIN pages of `sp` in one row group; no statistics in the second file)
REFUSALS = {
    "refuse_distinct": (["b"], [count_distinct("s")], [], {}),
    "refuse_median": (["b"], [median("x")], [], {}),
    "refuse_sp_like": (["sp"], [count_star()], [("sp_like", "v%")], {}),
    "refuse_minmax_sp_like": (["b"], [min_("sp")], [("sp_like", "v%")], {}),
}


def ts_bound(g: int) -> int:
    """The first timestamp of row group g (test_ranks_one_gpu.py lays the row groups out at these offsets)."""
    return 1_700_000_000_000 + g * 30 * HOUR


def filters_of(spec):
    out = []
    for kind, v in spec:
        if kind == "ts_lt":
            from parseable_b200.query import Timestamp
            out.append(col("ts") < Timestamp(ts_bound(v)))
        elif kind == "x_gt":
            out.append(col("x") > float(v))
        elif kind == "f_gt":
            out.append(col("f") > float(v))
        elif kind == "f_lt":
            out.append(col("f") < float(v))
        elif kind == "i_eq":
            out.append(col("i") == v)
        elif kind == "sp_like":
            out.append(col("sp").like(v))
        else:
            raise ValueError(kind)
    return out


def _write(out, name, res=None, err=None, seconds=0.0):
    import pyarrow as pa
    if err is not None:
        with open(out + ".json.tmp", "w") as f:
            json.dump({"code": err.code, "message": err.message, "seconds": seconds}, f)
        os.replace(out + ".json.tmp", out + ".json")
        return
    if res.json_text is not None:
        t = pa.table({"json": pa.array([res.json_text.decode()])})
    else:
        t = res.table()
    with pa.OSFile(out + ".arrow.tmp", "wb") as f, pa.ipc.new_file(f, t.schema) as w:
        w.write_table(t)
    os.replace(out + ".arrow.tmp", out + ".arrow")


def run_case(prov, case, out, flags):
    from parseable_b200.query import QueryError
    keys, aggs, flt, kw = case
    print(os.path.basename(out), flush=True)
    t0 = time.time()
    try:
        res = prov.aggregate(keys, aggs, filters_of(flt), flags=flags, **kw)
    except QueryError as e:
        _write(out, None, err=e, seconds=time.time() - t0)
        return False
    _write(out, None, res=res)
    return True


def join(lib, L, idfile, n, rank):
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
                raise SystemExit("timeout waiting for the communicator id")
            time.sleep(0.01)
        ident = open(idfile, "rb").read()
    assert lib.pq_comm_init_rank(ident, n, rank) == 0, lib.pq_last_error(None)


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
    cols = list(schema)
    AR = L.PQ_QUERY_ALLREDUCE

    def path(name, src):
        return os.path.join(out, f"{name}.{src}.{rank}")

    table = DeviceTable(files, cols, shard_index=rank, shard_count=n)
    provs = {"table": StandardTableProvider(table, schema=schema),
             "files": StandardTableProvider(files, schema=schema, shard_index=rank, shard_count=n)}
    for src, prov in provs.items():
        for name, case in CASES.items():
            run_case(prov, case, path(name, src), AR)
        for name in LOCAL:
            run_case(prov, CASES[name], path("local_" + name, src), 0)
        _write(path("local_rowids", src), None, res=prov.scan(filters=filters_of([("x_gt", 0)])))   # global __row_id
        # refusals, then the next query on the same communicator
        for name, case in REFUSALS.items():
            run_case(prov, case, path(name, src), AR)
            run_case(prov, CASES["fp_s"], path("after_" + name, src), AR)
    # DATE_BIN over a file list whose second file has no statistics: the ranks that read it refuse
    nostats = StandardTableProvider(spec["nostats"], schema=schema, shard_index=rank, shard_count=n)
    run_case(nostats, CASES["fp_bin"], path("refuse_bin_nostats", "files"), AR)
    run_case(provs["files"], CASES["fp_bin"], path("after_refuse_bin_nostats", "files"), AR)

    # the agreed key numbering is cached with the table: the same query twice, then after rank 1 alone reopens its
    # table, then on a new communicator (a new epoch)
    prov = provs["table"]
    seq = [("fp_s", "fp_s"), ("minmax_str_by_s", "minmax_str_by_s")]
    for step in ("again", "reopen", "epoch"):
        if step == "reopen" and rank == 1:
            table.close()
            table = DeviceTable(files, cols, shard_index=rank, shard_count=n)
            prov = StandardTableProvider(table, schema=schema)
        if step == "epoch":
            assert lib.pq_comm_destroy() == 0
            join(lib, L, spec["idfile"] + ".2", n, rank)
        for name, case in seq:
            run_case(prov, CASES[case], path(f"cache_{step}_{name}", "table"), AR)
    table.close()
    assert lib.pq_comm_destroy() == 0
    print(f"rank {rank}/{n}: done", flush=True)


if __name__ == "__main__":
    main()
