"""CPU tests of the pure host/device decode functions (decode_core.cuh) through the test-only
harness tools/libdecode_core_host.so.  The same source is compiled into the CUDA kernels."""
import ctypes as C
import os
import struct

import numpy as np
import pytest


@pytest.fixture(scope="module")
def dc(built):
    lib = C.CDLL(os.path.join(built, "tools", "libdecode_core_host.so"))
    lib.dc_decode_hybrid.restype = C.c_int64
    lib.dc_f64_key.restype = C.c_int64
    lib.dc_f64_key.argtypes = [C.c_uint64]
    lib.dc_f64_from_key.restype = C.c_uint64
    lib.dc_f64_from_key.argtypes = [C.c_int64]
    lib.dc_load_u64.restype = C.c_uint64
    return lib


def _uleb(v):
    out = bytearray()
    while True:
        b = v & 0x7F
        v >>= 7
        if v:
            out.append(b | 0x80)
        else:
            out.append(b)
            return bytes(out)


def encode_hybrid(values, bw, rng, rle_bias=0.5, min_rle=1):
    """Reference encoder for tests: random mix of RLE runs and bit-packed runs (Parquet
    'RLE/bit-packing hybrid'), including runs of 1 and long bit-packed runs with multi-byte headers."""
    out = bytearray()
    i, n = 0, len(values)
    while i < n:
        # length of the run of equal values at i
        j = i
        while j < n and values[j] == values[i]:
            j += 1
        run = j - i
        if run >= min_rle and rng.random() < rle_bias:
            take = int(rng.integers(1, run + 1))
            out += _uleb(take << 1)
            out += int(values[i]).to_bytes((bw + 7) // 8, "little")
            i += take
        else:
            groups = int(rng.integers(1, 80))
            take = min(groups * 8, n - i)
            groups = (take + 7) // 8
            chunk = list(values[i:i + take]) + [0] * (groups * 8 - take)
            out += _uleb((groups << 1) | 1)
            acc, nbits = 0, 0
            buf = bytearray()
            for v in chunk:
                acc |= int(v) << nbits
                nbits += bw
                while nbits >= 8:
                    buf.append(acc & 0xFF)
                    acc >>= 8
                    nbits -= 8
            assert nbits == 0
            out += buf
            i += take
    return bytes(out)


@pytest.mark.parametrize("bw", [0, 1, 2, 3, 5, 8, 11, 13, 16, 17, 24, 31, 32])
@pytest.mark.parametrize("pattern", ["random", "runs"])
def test_hybrid_roundtrip(dc, bw, pattern):
    rng = np.random.default_rng(bw * 7 + (pattern == "runs"))
    n = 9000
    hi = (1 << bw) if bw else 1
    if pattern == "random":
        vals = rng.integers(0, hi, n, dtype=np.uint64)
    else:
        vals = np.repeat(rng.integers(0, hi, n // 7 + 1, dtype=np.uint64), rng.integers(1, 40, n // 7 + 1))[:n]
    vals = vals.astype(np.uint64)
    enc = encode_hybrid(vals, bw, rng)
    out = np.zeros(n, np.uint32)
    # the kernel's real geometry
    slab = 2048
    cap = ((slab * bw // 8 + slab // 8 + 64 + 15) // 16) * 16
    got = dc.dc_decode_hybrid(enc, C.c_uint64(len(enc)), bw, n, slab, cap, 64, out.ctypes.data_as(C.c_void_p))
    assert got == n
    assert np.array_equal(out.astype(np.uint64), vals)


@pytest.mark.parametrize("bw,cap,max_ent", [(1, 64, 4), (3, 48, 2), (13, 160, 3), (7, 32, 64)])
def test_hybrid_tiny_windows_force_slab_shrink(dc, bw, cap, max_ent):
    """Windows / directories far smaller than a slab: the walker must stop early and resume without
    losing or duplicating values (the kernel's slab-shrink path)."""
    rng = np.random.default_rng(99 + bw)
    n = 5000
    vals = np.repeat(rng.integers(0, 1 << bw, n, dtype=np.uint64), rng.integers(1, 12, n))[:n]
    enc = encode_hybrid(vals, bw, rng, rle_bias=0.7)
    out = np.zeros(n, np.uint32)
    got = dc.dc_decode_hybrid(enc, C.c_uint64(len(enc)), bw, n, 2048, cap, max_ent, out.ctypes.data_as(C.c_void_p))
    assert got == n
    assert np.array_equal(out.astype(np.uint64), vals)


@pytest.mark.parametrize("pattern", ["random", "skewed", "long_runs", "mixed", "short_runs"])
@pytest.mark.parametrize("bw", [0, 1, 3, 6, 8, 9, 11, 14, 17])
def test_walker_directory_and_octet_pass_replica(dc, bw, pattern):
    """CPU replica of k_scan's per-slab walk and the octet pass (tools/decode_core_host.cpp): the
    selection bits of a dictionary-LUT leaf over one 20 000-row page must equal LUT[value] for every
    run structure — bit-packed only, a skewed column (many short runs), long RLE runs, a mix whose
    octets straddle directory entries, and RLE runs of 1-4 values, more than one directory holds, so
    that slabs shrink and later slabs start inside a byte or word of the bitmap."""
    rng = np.random.default_rng(100 * bw + len(pattern))
    n = 20000
    hi = (1 << bw) if bw else 1
    rle_bias = 0.5
    if pattern == "random":
        vals = rng.integers(0, hi, n, dtype=np.uint64)
    elif pattern == "skewed":
        vals = np.where(rng.random(n) < 0.8, 0, rng.integers(0, hi, n)).astype(np.uint64)
    elif pattern == "long_runs":
        vals = np.repeat(rng.integers(0, hi, n // 150 + 2, dtype=np.uint64), rng.integers(100, 400, n // 150 + 2))[:n]
    elif pattern == "mixed":
        vals = np.repeat(rng.integers(0, hi, n // 5 + 2, dtype=np.uint64), rng.integers(1, 30, n // 5 + 2))[:n]
    else:
        vals = np.repeat(rng.integers(0, hi, n // 2 + 2, dtype=np.uint64), rng.integers(1, 5, n // 2 + 2))[:n]
        rle_bias = 1.0
    vals = vals.astype(np.uint64)
    enc = encode_hybrid(vals, bw, rng, rle_bias=rle_bias)
    smem = 1 if hi <= 2048 else 0
    lut = (rng.random(max(hi, 2048)) < 0.3).astype(np.uint8)
    bitmap = np.zeros((n + 31) // 32 + 1, np.uint32)
    shrunk = C.c_uint32(0)
    dc.dc_walk_octet_scan.restype = C.c_int64
    got = dc.dc_walk_octet_scan(enc, C.c_uint64(len(enc)), bw, n, lut.ctypes.data_as(C.c_void_p), smem,
                                bitmap.ctypes.data_as(C.c_void_p), C.byref(shrunk))
    assert got == n
    exp = np.packbits(lut[vals.astype(np.int64)].astype(bool), bitorder="little")
    assert np.array_equal(bitmap.view(np.uint8)[: len(exp)], exp), (bw, pattern, shrunk.value)
    if pattern == "long_runs" and bw >= 1:
        assert shrunk.value == 0    # a handful of long runs per slab fits one directory
    if pattern == "short_runs" and bw >= 1:
        assert shrunk.value >= 1    # the octet pass runs over shrunk slabs


def test_f64_order_key_is_total_order(dc):
    vals = [float("-inf"), -1e300, -1.5, -0.0, 0.0, 5e-324, 1.5, 1e300, float("inf")]
    nan_pos = struct.unpack("<d", struct.pack("<Q", 0x7FF8000000000001))[0]
    nan_neg_bits = 0xFFF8000000000001
    keys = [dc.dc_f64_key(struct.unpack("<Q", struct.pack("<d", v))[0]) for v in vals]
    assert keys == sorted(keys) and len(set(keys)) == len(keys)
    k_nan = dc.dc_f64_key(struct.unpack("<Q", struct.pack("<d", nan_pos))[0])
    assert k_nan > keys[-1]                                  # +NaN greatest
    assert dc.dc_f64_key(nan_neg_bits) < keys[0]             # -NaN smallest
    for v in vals:
        b = struct.unpack("<Q", struct.pack("<d", v))[0]
        assert dc.dc_f64_from_key(dc.dc_f64_key(b)) == b


def test_unaligned_loads(dc):
    raw = bytes(range(1, 65))
    buf = C.create_string_buffer(raw, 80)
    base = C.addressof(buf)
    for off in range(0, 40):
        want = int.from_bytes(raw[off:off + 8], "little")
        assert dc.dc_load_u64(C.c_void_p(base), off) == want


LIKE_CASES = [
    (b"hello world", b"hello world", 0, False, True), (b"hello", b"hell", 0, False, False),
    (b"hello world", b"hello", 1, False, True), (b"hello world", b"world", 2, False, True),
    (b"a timeout-xyzzy b", b"timeout-xyzzy", 3, False, True), (b"abc", b"", 3, False, True),
    (b"Hello", b"hello", 0, True, True), (b"abc", b"a_c", 4, False, True), (b"abbc", b"a_c", 4, False, False),
    (b"a%c", b"a\\%c", 4, False, True), (b"abc", b"a\\%c", 4, False, False), (b"xaybzc", b"%a%b%c", 4, False, True),
    (b"xaybz", b"%a%b%c", 4, False, False), ("héllo".encode(), "h_llo".encode(), 4, False, True),
    (b"", b"%", 4, False, True), (b"", b"_", 4, False, False),
]


@pytest.mark.parametrize("s,p,kind,ci,want", LIKE_CASES)
def test_like_match(dc, s, p, kind, ci, want):
    assert bool(dc.dc_like(s, len(s), p, len(p), kind, int(ci))) == want


def test_device_like_matcher_agrees_with_acero(dc):
    """like_general is the very function k_leaf_luts runs per dictionary entry (host/device code): every
    (value, pattern) pair of a grid with wildcards, escapes, empty strings and multi-byte characters
    must agree with Acero's match_like; ILIKE is compared on ASCII patterns (the matcher folds ASCII only)."""
    import pyarrow as pa
    import pyarrow.compute as pc
    vals = ["", "a", "ab", "abc", "a%c", "a_c", "A_C", "abcabc", "xxabcxx", "ABC", "aXc", "%", "_", "a\\c", "timeout", "Timeout after 30s",
            "GET /api/v1/users/42", "get /api/v1/users/42", "ééé", "aéc", "日本語ログ", "a\nb"]
    pats = ["%", "", "a", "a%", "%c", "%b%", "a_c", "a\\_c", "a\\%c", "%\\%%", "_", "__", "___", "%abc%abc%", "abc%abc", "%a%b%c%", "A_C", "%timeout%",
            "Timeout%30s", "GET /api/%/users/__", "a%c", "%é%", "a_c%", "%_", "_%_", "日_語%", "%\\\\%"]
    arr = pa.array(vals, pa.string())
    for p in pats:
        pb = p.encode()
        for ci in (False, True):
            if ci and any(ord(ch) > 127 for ch in p):
                continue
            want = pc.match_like(arr, p, ignore_case=ci).to_pylist()
            for v, w in zip(vals, want):
                if ci and any(ord(ch) > 127 for ch in v):
                    continue
                vb = v.encode()
                assert bool(dc.dc_like(vb, len(vb), pb, len(pb), 4, int(ci))) == w, (v, p, ci)


def _page_payloads(path, col):
    """Raw data-page payloads of column `col` (row group 0) located with the library's own page walk."""
    import ctypes as C
    import json
    from parseable_b200 import _lib as L
    lib = L.load()
    f = L.PqFile(path=path.encode())
    n = lib.pq_file_describe(C.byref(f), None, 0)
    buf = C.create_string_buffer(n + 1)
    lib.pq_file_describe(C.byref(f), buf, n + 1)
    d = json.loads(buf.value.decode())
    cc = d["row_groups"][0]["columns"][col]
    off = cc["dictionary_page_offset"] if 0 < cc["dictionary_page_offset"] < cc["data_page_offset"] else cc["data_page_offset"]
    raw = open(path, "rb").read()
    out = []
    for p in cc["pages"]:
        start = off + p["header_len"]
        if p["type"] in (0, 3):
            out.append((raw[start:start + p["compressed_size"]], p["num_values"], p["encoding"]))
        off = start + p["compressed_size"]
    return out


@pytest.mark.parametrize("kind", ["timestamps", "random_wide", "constant", "negative_steps"])
def test_delta_binary_packed_pages_from_pyarrow(dc, built, tmp_path, kind):
    """DELTA_BINARY_PACKED pages written by pyarrow (an independent encoder) decode to the source values
    through walk_delta / bp_get64 with the kernel's slab and window geometry."""
    import pyarrow as pa
    import pyarrow.parquet as pq
    rng = np.random.default_rng(11)
    n = 50_000
    if kind == "timestamps":
        vals = (1_700_000_000_000 - np.cumsum(rng.integers(0, 3, n) * rng.integers(1, 50, n))).astype(np.int64)
    elif kind == "random_wide":
        vals = rng.integers(-2**62, 2**62, n, dtype=np.int64)
    elif kind == "constant":
        vals = np.full(n, 42, np.int64)
    else:
        vals = np.cumsum(rng.integers(-1000, 5, n)).astype(np.int64)
    path = str(tmp_path / f"delta_{kind}.parquet")
    t = pa.table({"v": pa.array(vals)}).cast(pa.schema([pa.field("v", pa.int64(), False)]))
    pq.write_table(t, path, compression="NONE", use_dictionary=False, column_encoding={"v": "DELTA_BINARY_PACKED"},
                   data_page_size=1 << 20, max_rows_per_page=20_000)
    dc.dc_decode_delta.restype = C.c_int64
    pos = 0
    for payload, nv, enc in _page_payloads(path, 0):
        assert enc == 5
        out = np.zeros(nv, np.int64)
        for cap in (8192 + 64, 640):                     # the kernel's window, and a tiny one that forces resumes
            got = dc.dc_decode_delta(payload, C.c_uint64(len(payload)), nv, 2048, cap, 80, out.ctypes.data_as(C.c_void_p))
            assert got == nv, (kind, cap, got)
            assert np.array_equal(out, vals[pos:pos + nv]), (kind, cap)
        pos += nv
    assert pos == n
