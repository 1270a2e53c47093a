"""No-GPU tests of the host metadata layer and of the C-ABI surface: the library loads, exports
every symbol include/parseable_b200.h declares, and its footer / page-header reader agrees with
pyarrow's independent reader on the synthetic Parseable-style files and the golden fixtures."""
import ctypes as C
import json
import os
import re

import pyarrow.parquet as pq
import pytest

from parseable_b200 import _lib as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib(built):
    return L.load()


def describe(lib, path):
    f = L.PqFile(path=path.encode())
    n = lib.pq_file_describe(C.byref(f), None, 0)
    assert n > 0, lib.pq_last_error(None)
    buf = C.create_string_buffer(n + 1)
    assert lib.pq_file_describe(C.byref(f), buf, n + 1) == n
    return json.loads(buf.value.decode())


def test_exports_match_header(lib):
    hdr = open(os.path.join(ROOT, "include", "parseable_b200.h")).read()
    declared = set(re.findall(r"\b(pq_[a-z_0-9]+)\s*\(", hdr))
    assert declared == set(L.EXPORTS)
    for name in declared:
        assert hasattr(lib, name), name
    assert b"sm_90a" in lib.pq_version()


def test_struct_layouts_match_header(lib, tmp_path):
    """The header is valid plain C and the ctypes mirror has the same struct sizes gcc computes."""
    import subprocess
    src = tmp_path / "sizes.c"
    src.write_text('#include <stdio.h>\n#include "parseable_b200.h"\nint main(void){printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu\\n",'
                   'sizeof(PqLiteral),sizeof(PqPredOp),sizeof(PqAgg),sizeof(PqFile),sizeof(PqColumn),sizeof(PqQueryDesc),'
                   'sizeof(PqMetrics),sizeof(struct ArrowArray),sizeof(struct ArrowSchema),sizeof(PqPlanFilter),sizeof(PqColumnStat),'
                   'sizeof(PqManifestFile),sizeof(PqManifestItem),sizeof(PqTimeBound));return 0;}\n')
    exe = tmp_path / "sizes"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    sizes = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    mirror = [L.PqLiteral, L.PqPredOp, L.PqAgg, L.PqFile, L.PqColumn, L.PqQueryDesc, L.PqMetrics, L.ArrowArray, L.ArrowSchema,
              L.PqPlanFilter, L.PqColumnStat, L.PqManifestFile, L.PqManifestItem, L.PqTimeBound]
    assert sizes == [C.sizeof(m) for m in mirror]


def test_no_device_is_an_error_not_a_fallback(lib):
    if lib.pq_device_count() > 0:
        pytest.skip("a GPU is present")
    rc = lib.pq_init(None, 0)
    assert rc == L.PQ_ERR_CUDA
    assert b"CUDA" in lib.pq_last_error(None)
    d = L.PqQueryDesc()
    h = C.c_void_p()
    assert lib.pq_query_open(C.byref(d), C.byref(h)) == L.PQ_ERR_CUDA


def check_against_pyarrow(lib, path):
    d = describe(lib, path)
    md = pq.ParquetFile(path).metadata
    assert d["num_rows"] == md.num_rows
    assert len(d["row_groups"]) == md.num_row_groups
    assert [l["name"] for l in d["leaves"]] == [md.schema.column(i).path for i in range(md.num_columns)]
    for l, i in zip(d["leaves"], range(md.num_columns)):
        c = md.schema.column(i)
        assert l["max_def"] == c.max_definition_level and l["max_rep"] == c.max_repetition_level
    for g in range(md.num_row_groups):
        rg = md.row_group(g)
        assert d["row_groups"][g]["num_rows"] == rg.num_rows
        for c in range(rg.num_columns):
            cc, dc = rg.column(c), d["row_groups"][g]["columns"][c]
            assert dc["num_values"] == cc.num_values
            assert dc["total_uncompressed_size"] == cc.total_uncompressed_size
            assert dc["total_compressed_size"] == cc.total_compressed_size
            assert dc["data_page_offset"] == cc.data_page_offset
            if cc.has_dictionary_page:
                assert dc["dictionary_page_offset"] == cc.dictionary_page_offset
            if cc.statistics is not None and cc.statistics.has_null_count:
                assert dc["null_count"] == cc.statistics.null_count
            pages = dc["pages"]
            # headers + payloads tile the chunk exactly; data pages carry all the values
            assert sum(p["header_len"] + p["compressed_size"] for p in pages) == cc.total_compressed_size
            assert sum(p["num_values"] for p in pages if p["type"] in (0, 3)) == cc.num_values
            assert sum(1 for p in pages if p["type"] == 2) == (1 if cc.has_dictionary_page else 0)
    return d


def test_describe_synthetic(lib, small_files):
    d = check_against_pyarrow(lib, small_files["nulls"])
    # Parseable writer shape: p_timestamp DELTA_BINARY_PACKED (5), others RLE_DICTIONARY (8) with
    # PLAIN (0) fallback; 20 000-row pages
    cols = d["row_groups"][0]["columns"]
    assert all(p["encoding"] == 5 for p in cols[0]["pages"])
    assert {p["encoding"] for p in cols[1]["pages"] if p["type"] == 0} == {8}
    assert {p["encoding"] for p in cols[4]["pages"] if p["type"] == 0} <= {0, 8}
    assert max(p["num_values"] for p in cols[1]["pages"] if p["type"] == 0) == 20000


def test_describe_golden(lib):
    for f in ("field_stats_10rows.parquet", "field_stats_1000rows.parquet", "field_stats_empty.parquet"):
        check_against_pyarrow(lib, os.path.join(ROOT, "tests", "golden", f))


def test_corrupt_and_missing_files(lib, tmp_path):
    f = L.PqFile(path=str(tmp_path / "nope.parquet").encode())
    assert lib.pq_file_describe(C.byref(f), None, 0) == L.PQ_ERR_IO
    bad = tmp_path / "bad.parquet"
    bad.write_bytes(b"PAR1" + b"\x00" * 64 + b"PAR1")
    f = L.PqFile(path=str(bad).encode())
    assert lib.pq_file_describe(C.byref(f), None, 0) == L.PQ_ERR_CORRUPT
    trunc = tmp_path / "trunc.parquet"
    good = open(os.path.join(ROOT, "tests", "golden", "field_stats_10rows.parquet"), "rb").read()
    trunc.write_bytes(good[: len(good) // 2])
    f = L.PqFile(path=str(trunc).encode())
    assert lib.pq_file_describe(C.byref(f), None, 0) == L.PQ_ERR_CORRUPT
