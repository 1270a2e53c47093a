"""The ZSTD and GZIP page decoders (parseable_b200/csrc/zstd_decode.cuh, inflate_decode.cuh) compiled for the host -- the same source the GPU
runs with 32 lanes -- against pyarrow's zstd: every block / literals / sequence mode the encoder emits at its levels,
multi-block inputs, empty and one-byte pages, Parquet pages out of a zstd file, and garbled input (no fault).
ZSTD is a legal P_PARQUET_COMPRESSION_ALGO of the reference (src/option.rs:62-86)."""
import ctypes
import os
import subprocess

import numpy as np
import pyarrow as pa
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def zs():
    so = os.path.join(ROOT, "tools", "libzstd_host.so")
    if not os.path.exists(so):
        subprocess.check_call(["make", "-C", ROOT, "tools"])
    lib = ctypes.CDLL(so)
    for f in (lib.zs_host_decode, lib.gz_host_decode):
        f.argtypes = [ctypes.c_void_p, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_uint64]
        f.restype = ctypes.c_int

    def decode(comp: bytes, n: int, gz: bool = False):
        src = np.frombuffer(comp, dtype=np.uint8).copy() if comp else np.zeros(1, np.uint8)
        dst = np.zeros(max(n, 1), np.uint8)
        ok = (lib.gz_host_decode if gz else lib.zs_host_decode)(src.ctypes.data, len(comp), dst.ctypes.data, n)
        return ok == 1, dst[:n].tobytes()
    return decode


def _inputs():
    rng = np.random.default_rng(11)
    words = [b"request", b"completed", b"failed", b"retry", b"upstream", b"cache", b"miss", b"hit", b"db", b"query"]
    yield "empty", b""
    yield "one", b"x"
    yield "text", b"the quick brown fox jumps over the lazy dog. " * 4000
    yield "random", rng.integers(0, 256, 300_000, dtype=np.uint8).tobytes()           # raw blocks
    yield "zeros", bytes(500_000)                                                       # RLE blocks
    yield "skewed", rng.choice(np.frombuffer(b"abcdefgh", np.uint8), 400_000,
                               p=[.5, .2, .1, .08, .05, .04, .02, .01]).tobytes()       # Huffman literals, 4 streams
    yield "i64", np.cumsum(rng.integers(0, 50, 100_000)).astype(np.int64).tobytes()
    yield "f64_dict", (np.floor(rng.lognormal(3.5, 1.2, 100_000)) / 1000.0).tobytes()
    yield "logs", b"".join(b"[%04d] " % rng.integers(0, 8192) + b" ".join(words[j] for j in rng.integers(0, 10, rng.integers(3, 8))) + b"\n"
                           for _ in range(20_000))
    idx = rng.choice(5, size=800_000, p=[.3, .55, .09, .05, .01]).astype(np.uint8)
    yield "bitpacked3", np.packbits(((idx[:, None] >> np.arange(3)) & 1).astype(np.uint8), bitorder="little").tobytes()
    yield "short_repeats", (b"ab" * 7 + b"c") * 3000


@pytest.mark.parametrize("level", [None, -5, 1, 3, 9, 19, 22])
def test_decoder_matches_zstd(zs, level):
    for name, data in _inputs():
        codec = pa.Codec("zstd") if level is None else pa.Codec("zstd", compression_level=level)
        comp = codec.compress(data, asbytes=True)
        ok, out = zs(comp, len(data))
        assert ok and out == data, (name, level, len(data), len(comp))


def test_concatenated_and_skippable_frames(zs):
    a, b = b"hello " * 1000, bytes(range(256)) * 40
    c = pa.Codec("zstd")
    comp = c.compress(a, asbytes=True) + b"\x50\x2a\x4d\x18\x03\x00\x00\x00abc" + c.compress(b, asbytes=True)
    ok, out = zs(comp, len(a) + len(b))
    assert ok and out == a + b


def test_wrong_size_and_garbled_input_are_refused_without_faults(zs):
    rng = np.random.default_rng(5)
    data = b"".join(b"%d,%d;" % (i % 97, i * i % 1013) for i in range(40_000))
    comp = pa.Codec("zstd", compression_level=3).compress(data, asbytes=True)
    assert not zs(comp, len(data) - 1)[0]
    assert not zs(comp, len(data) + 1)[0]
    assert not zs(comp[:-5], len(data))[0]
    assert not zs(b"\x00" * 16, 10)[0]
    refused = 0
    for _ in range(300):
        g = bytearray(comp)
        for _ in range(int(rng.integers(1, 4))):
            g[int(rng.integers(0, len(g)))] ^= 1 << int(rng.integers(0, 8))
        ok, out = zs(bytes(g), len(data))     # content checksums are not verified: a flip inside literals may pass
        refused += 0 if ok else 1
    assert refused > 50


def test_pages_of_a_zstd_parquet_file(zs, tmp_path, built):
    """The page payloads as the table-open path cuts them (csrc/table.cu, through pq_file_describe's page walk):
    compressed_size bytes behind every page header decode to uncompressed_size bytes, equal to the payload of the same
    page of the same file written uncompressed."""
    import ctypes as C
    import json
    from parseable_b200 import _lib as L
    from parseable_b200 import synth
    lib = L.load()

    def describe(path):
        f = L.PqFile(path=path.encode())
        n = lib.pq_file_describe(C.byref(f), None, 0)
        assert n > 0
        buf = C.create_string_buffer(n + 1)
        lib.pq_file_describe(C.byref(f), buf, n + 1)
        return json.loads(buf.value.decode())

    def payloads(path):
        raw = open(path, "rb").read()
        out = []
        for col in describe(path)["row_groups"][0]["columns"]:
            start = col["dictionary_page_offset"] if 0 < col["dictionary_page_offset"] < col["data_page_offset"] else col["data_page_offset"]
            pos = start
            for pg in col["pages"]:
                pos += pg["header_len"]
                out.append((col["codec"], pg, raw[pos:pos + pg["compressed_size"]]))
                pos += pg["compressed_size"]
        return out
    pz, pn = str(tmp_path / "z.parquet"), str(tmp_path / "n.parquet")
    cols = ["level", "host", "latency_ms", "cpu", "message"]
    synth.write_logs16(pz, n_row_groups=1, rows_per_group=50_000, compression="ZSTD", columns=cols)
    synth.write_logs16(pn, n_row_groups=1, rows_per_group=50_000, compression="NONE", columns=cols)
    zp, np_ = payloads(pz), payloads(pn)
    assert len(zp) == len(np_) >= 2 * len(cols)
    for (codec, pg, comp), (_, png, want) in zip(zp, np_):
        assert codec == 6 and pg["uncompressed_size"] == len(want) == png["uncompressed_size"]
        ok, out = zs(comp, pg["uncompressed_size"])
        assert ok and out == want


# ---- GZIP (codec 2): gzip members around DEFLATE ----
@pytest.mark.parametrize("level", [1, 6, 9])
def test_gzip_decoder_matches_zlib(zs, level):
    import gzip
    import zlib
    for name, data in _inputs():
        for how in ("arrow", "gzip", "fixed", "stored+members"):
            if how == "arrow":
                comp = pa.Codec("gzip", compression_level=level).compress(data, asbytes=True)
            elif how == "gzip":
                comp = gzip.compress(data, compresslevel=level)
            elif how == "fixed":                       # fixed Huffman blocks only
                co = zlib.compressobj(level, zlib.DEFLATED, 31, 9, zlib.Z_FIXED)
                comp = co.compress(data) + co.flush()
            else:                                      # stored blocks, then a second member
                h = len(data) // 2
                comp = gzip.compress(data[:h], compresslevel=0) + gzip.compress(data[h:], compresslevel=level)
            ok, out = zs(comp, len(data), gz=True)
            assert ok and out == data, (name, level, how, len(data), len(comp))


def test_gzip_garbled_input_is_refused_without_faults(zs):
    import gzip
    rng = np.random.default_rng(9)
    data = b"".join(b"%d,%d;" % (i % 97, i * i % 1013) for i in range(40_000))
    comp = gzip.compress(data, compresslevel=6)
    assert not zs(comp, len(data) - 1, gz=True)[0] and not zs(comp, len(data) + 1, gz=True)[0]
    assert not zs(comp[:-9], len(data), gz=True)[0] and not zs(b"\x00" * 32, 10, gz=True)[0]
    refused = 0
    for _ in range(300):
        g = bytearray(comp)
        for _ in range(int(rng.integers(1, 4))):
            g[int(rng.integers(0, len(g)))] ^= 1 << int(rng.integers(0, 8))
        refused += 0 if zs(bytes(g), len(data), gz=True)[0] else 1     # CRC-32 is not verified: a flip inside literals may pass
    assert refused > 50


# ---- the same inputs through the GPU kernels (k_decompress_zstd: 32 lanes, four Huffman streams on lanes 0-3,
# persistent warps taking pages by ticket) -- one launch per test, every page at its own source phase ----
@pytest.mark.gpu
def test_gpu_zstd_levels():
    from test_page_codecs import ZSTD, DevImages
    im = DevImages()
    for li, level in enumerate([None, -5, 1, 3, 9, 19, 22]):
        codec = pa.Codec("zstd") if level is None else pa.Codec("zstd", compression_level=level)
        for k, (name, data) in enumerate(_inputs()):
            im.add(ZSTD, codec.compress(data, asbytes=True), data, sphase=(li + k) % 16, odd=k % 2 == 1)
    dst, flag = im.run()
    assert flag == 0
    im.check(dst)


@pytest.mark.gpu
def test_gpu_gzip_variants():
    import gzip
    import zlib
    from test_page_codecs import GZIP, DevImages
    im = DevImages()
    for li, level in enumerate([1, 6, 9]):
        for k, (name, data) in enumerate(_inputs()):
            h = len(data) // 2
            co = zlib.compressobj(level, zlib.DEFLATED, 31, 9, zlib.Z_FIXED)
            for v, comp in enumerate((pa.Codec("gzip", compression_level=level).compress(data, asbytes=True),
                                      gzip.compress(data, compresslevel=level),
                                      co.compress(data) + co.flush(),
                                      gzip.compress(data[:h], compresslevel=0) + gzip.compress(data[h:], compresslevel=level))):
                im.add(GZIP, comp, data, sphase=(li + k + v) % 16, odd=(k + v) % 2 == 1)
    dst, flag = im.run()
    assert flag == 0
    im.check(dst)
