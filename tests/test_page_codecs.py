"""The LZ4_RAW, SNAPPY and stored page decoders (parseable_b200/csrc/lz_decode.cuh) byte for byte against pyarrow's
codecs, and the kernels that run them and the ZSTD / GZIP decoders on the GPU (decomp_kernels.cuh).

On the CPU the decoders are compiled for the host with every copy run lane by lane for all 32 lanes, once in ascending
and once in descending lane order (tools/lz_host.cpp).  They are checked on:
  - pyarrow's encodings of the corpus of test_zstd.py;
  - hand-built streams that reach every token form: LZ4 length extensions ending in 0 and in 255, match offsets 1-31
    (the source overlaps the copying lanes), Snappy copy-1 / copy-2 / copy-4 tags and literals with 1-4 length bytes,
    and literals whose lengths reach the head, the tail and the 4x-unrolled loop of the funnel-shift copy -- each
    stream at source and destination phases 0-15;
  - a table of malformed streams, each refused, including a Snappy literal length that wraps 32 bits;
  - a few hundred bit flips per format: canaries on both sides of the destination stay untouched, and where pyarrow
    accepts a stream the decoder gives the same bytes.
The malformed and garbled cases run in a child process, so that a decoder that writes out of bounds fails its test
instead of ending the run.  The GPU tests launch the kernels through the same launch_decompress as the table-open path
(tools/decomp_dev.cu)."""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pyarrow as pa
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_zstd import _inputs  # noqa: E402

LZ4, SNAPPY, STORED, ZSTD, GZIP = 7, 1, 0, 6, 2
GUARD = 64
CANARY = np.array([(i * 151 + 7) & 0xFF for i in range(GUARD)], np.uint8)
FILL = 0x5A   # what the destination holds before decoding


def _so(name):
    so = os.path.join(ROOT, "tools", name)
    if not os.path.exists(so):
        subprocess.check_call(["make", "-C", ROOT, "tools"])
    return so


class HostLz:
    """lz_host_decode of one build (lanes ascending or descending)."""

    def __init__(self, descending=False):
        self.lib = ctypes.CDLL(_so("liblz_host_desc.so" if descending else "liblz_host.so"))
        self.lib.lz_host_decode.argtypes = [ctypes.c_uint32, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_void_p,
                                            ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32]
        self.lib.lz_host_decode.restype = ctypes.c_int

    def __call__(self, codec, stream, n, sphase=0, dphase=0):
        """(accepted, the n destination bytes, canaries intact)"""
        src = np.frombuffer(stream, np.uint8).copy() if stream else np.zeros(1, np.uint8)
        out = np.full(2 * GUARD + n, FILL, np.uint8)
        out[:GUARD] = CANARY
        out[GUARD + n:] = CANARY[::-1]
        r = self.lib.lz_host_decode(codec, src.ctypes.data, len(stream), sphase, out.ctypes.data, n, dphase, GUARD)
        assert r >= 0, "harness: bad arguments"
        intact = np.array_equal(out[:GUARD], CANARY) and np.array_equal(out[GUARD + n:], CANARY[::-1])
        return r == 1, out[GUARD:GUARD + n].tobytes(), intact


_PA = {LZ4: pa.Codec("lz4_raw"), SNAPPY: pa.Codec("snappy")}


def reference(codec, stream, n):
    """pyarrow's verdict on `stream` decoding to exactly n bytes, and its output.  pyarrow takes an output size and
    accepts a stream that decodes to fewer bytes, so exactly n means: it decodes into n bytes and not into n - 1."""
    def run(m):
        try:
            return _PA[codec].decompress(stream, decompressed_size=m, asbytes=True)
        except (pa.ArrowException, OSError, ValueError):
            return None
    out = run(n)
    if out is None or (n and run(n - 1) is not None):
        return False, None
    return True, out


# ---- a plain encoder for both formats -------------------------------------------------------------------------------
# A stream is a list of ops: ("L", literal bytes) and ("M", offset, length), with LZ77 overlap semantics.
def expand(ops):
    out = bytearray()
    for op in ops:
        if op[0] == "L":
            out += op[1]
        else:
            _, off, ln = op
            assert 0 < off <= len(out)
            for _ in range(ln):
                out.append(out[-off])
    return bytes(out)


def _lz4_ext(n):
    return b"\xff" * (n // 255) + bytes([n % 255])


def lz4_encode(ops):
    """LZ4 block: ops alternate literal (maybe empty) and match, and end with a literal run (>= 16 bytes keeps the
    format's end rules: the last five bytes are literals and the last match starts 12 bytes before the end).
    Adjacent literal ops merge into one run."""
    merged = []
    for op in ops:
        if op[0] == "L" and merged and merged[-1][0] == "L":
            merged[-1] = ("L", merged[-1][1] + op[1])
        else:
            merged.append(op)
    ops = merged
    out = bytearray()
    i = 0
    while i < len(ops):
        lit = ops[i][1] if ops[i][0] == "L" else b""
        i += ops[i][0] == "L"
        m = ops[i] if i < len(ops) else None
        i += m is not None
        ml = m[2] - 4 if m else 0
        assert not m or m[2] >= 4
        out.append((min(len(lit), 15) << 4) | min(ml, 15))
        if len(lit) >= 15:
            out += _lz4_ext(len(lit) - 15)
        out += lit
        if m:
            out += m[1].to_bytes(2, "little")
            if ml >= 15:
                out += _lz4_ext(ml - 15)
    return bytes(out)


def _varint(v):
    out = bytearray()
    while v >= 0x80:
        out.append((v & 0x7F) | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


def snappy_encode(ops):
    """Snappy: a literal op may carry its count of length bytes ("L", data, nb) -- 0 inline, 1-4 extra bytes -- and a
    match op its tag kind ("M", off, len, kind) -- 1, 2 or 4 offset bytes."""
    out = bytearray(_varint(len(expand([op[:3] if op[0] == "M" else op[:2] for op in ops]))))
    for op in ops:
        if op[0] == "L":
            data = op[1]
            nb = op[2] if len(op) > 2 else (0 if len(data) <= 60 else ((len(data) - 1).bit_length() + 7) // 8)
            if nb == 0:
                out.append((len(data) - 1) << 2)
            else:
                out.append((59 + nb) << 2)
                out += (len(data) - 1).to_bytes(nb, "little")
            out += data
        else:
            _, off, ln, kind = op
            if kind == 1:
                assert 4 <= ln <= 11 and off < 2048
                out += bytes([1 | ((ln - 4) << 2) | ((off >> 8) << 5), off & 0xFF])
            elif kind == 2:
                assert 1 <= ln <= 64 and off < 65536
                out += bytes([2 | ((ln - 1) << 2)]) + off.to_bytes(2, "little")
            else:
                assert 1 <= ln <= 64
                out += bytes([3 | ((ln - 1) << 2)]) + off.to_bytes(4, "little")
    return bytes(out)


# literal lengths around the copy's 16-byte head and tail, its single-chunk loop (fewer than 97 chunks for lane 0) and
# its 4x-unrolled loop (128 chunks a trip, the remainder for some lanes only)
LIT_LENS = [1, 2, 3, 7, 15, 16, 17, 18, 31, 32, 33, 47, 48, 63, 64, 100, 255, 256, 271, 510, 1024, 1551, 1552, 1553, 1567,
            1568, 1584, 2047, 2048, 2064, 3100, 4109, 8191]


def _rand(rng, n):
    return rng.integers(0, 256, n, dtype=np.uint8).tobytes()


def lz4_streams():
    """name -> (stream, decoded bytes), every LZ4 token form"""
    rng = np.random.default_rng(71)
    tail = ("L", b"end of the block, literals only")
    cases = {}
    # literal lengths whose extension ends in 0 (15 + 255k) or carries a 255 byte (270 + ...)
    cases["lit_ext"] = [op for n in (1, 0, 14, 15, 16, 254, 269, 270, 271, 524, 525, 1000) for op in (("L", _rand(rng, n)), ("M", 1, 5))] + [tail]
    # match lengths: token only, extension ending in 0, carrying 255s
    cases["match_ext"] = [("L", _rand(rng, 40))] + [op for ml in (4, 5, 18, 19, 20, 273, 274, 275, 528, 529, 2000) for op in (("M", 17, ml), ("L", _rand(rng, 2)))] + [tail]
    # offsets 1-31: the match source overlaps the 32 lanes of the copy
    ops = [("L", _rand(rng, 64))]
    for off in range(1, 32):
        for ml in (4, off, off + 1, 31, 32, 33, 64, 100):
            if ml >= 4:
                ops += [("M", off, ml), ("L", _rand(rng, int(rng.integers(0, 3))))]
    cases["short_offsets"] = ops + [tail]
    # offsets 32 .. 65535, the largest a block can hold
    cases["long_offsets"] = [("L", _rand(rng, 66_000))] + [op for off in (32, 33, 64, 255, 256, 1000, 4096, 65535) for op in (("M", off, 40), ("L", b"."))] + [tail]
    # literal lengths for every part of the funnel-shift copy, each after a match so its phase moves
    cases["literal_copy"] = [("L", _rand(rng, 5))] + [op for n in LIT_LENS for op in (("M", 5, 4 + n % 7), ("L", _rand(rng, n)))] + [tail]
    cases["only_literals"] = [("L", _rand(rng, 5000))]
    out = {k: (lz4_encode(v), expand(v)) for k, v in cases.items()}
    out["empty"] = (b"\x00", b"")
    return out


def snappy_streams():
    rng = np.random.default_rng(73)
    cases = {}
    # literals with inline lengths 1-60 and 1-4 length bytes (also for short literals: the format allows it)
    cases["literal_lengths"] = [("L", _rand(rng, n)) for n in (1, 2, 59, 60, 61, 62, 255, 256, 257, 300, 65536, 65537)] + \
        [("L", _rand(rng, n), nb) for nb in (1, 2, 3, 4) for n in (1, 7, 33, 200)]
    cases["literal_copy"] = [op for n in LIT_LENS for op in (("L", _rand(rng, n)), ("M", 1, 4 + n % 8, 1))]
    # copy-1 (lengths 4-11, offsets < 2048), copy-2 (lengths 1-64) and copy-4 tags; offsets 1-31 overlap the lanes
    ops = [("L", _rand(rng, 3000))]
    for off in list(range(1, 32)) + [32, 33, 255, 256, 2047]:
        for ln in (4, 5, 8, 11):
            ops.append(("M", off, ln, 1))
        for ln in (1, 2, 3, 4, off, 32, 33, 64):
            if 1 <= ln <= 64:
                ops += [("M", off, ln, 2), ("M", off, ln, 4)]
        ops.append(("L", _rand(rng, 1)))
    cases["copies"] = ops
    cases["far_copies"] = [("L", _rand(rng, 70_000))] + [op for off in (2048, 65535, 65536, 69_999) for op in
                                                         (("M", off, 64, 4), ("M", off, 17, 2 if off < 65536 else 4), ("L", b"+"))]
    out = {k: (snappy_encode(v), expand([op[:3] if op[0] == "M" else op[:2] for op in v])) for k, v in cases.items()}
    out["empty"] = (b"\x00", b"")
    return out


def _malformed():
    """(codec, name, stream, dn): every one must be refused"""
    ok_lz = lz4_encode([("L", b"abcdefgh"), ("M", 8, 20), ("L", b"0123456789abcdefXYZ")])
    ok_sn = snappy_encode([("L", b"abcdefgh"), ("M", 8, 20, 2), ("L", b"0123456789")])
    n_lz, n_sn = len(expand([("L", b"abcdefgh"), ("M", 8, 20), ("L", b"0123456789abcdefXYZ")])), 38
    lit20 = bytes([19 << 2]) + b"A" * 20
    cases = [
        (LZ4, "offset_zero", bytes([0x40]) + b"abcd" + b"\x00\x00" + bytes([0x50]) + b"12345", 13),
        (LZ4, "offset_zero_first", bytes([0x00, 0x00, 0x00]) + bytes([0x50]) + b"12345", 9),
        (LZ4, "offset_past_output", bytes([0x40]) + b"abcd" + b"\x05\x00" + bytes([0x50]) + b"12345", 13),
        (LZ4, "lit_ext_missing", bytes([0xF0]), 15),
        (LZ4, "lit_ext_truncated_255", bytes([0xF0, 0xFF]), 300),
        (LZ4, "offset_truncated", bytes([0x40]) + b"abcd" + b"\x01", 8),
        (LZ4, "match_ext_missing", bytes([0x4F]) + b"abcd" + b"\x01\x00", 23),
        (LZ4, "match_ext_truncated_255", bytes([0x4F]) + b"abcd" + b"\x01\x00\xff", 300),
        (LZ4, "literal_past_source", bytes([0x50]) + b"abc", 5),
        (LZ4, "literal_ext_past_source", bytes([0xF0, 0x10]) + b"x" * 20, 31),
        (LZ4, "output_past_dn", ok_lz, n_lz - 1),
        (LZ4, "output_short_of_dn", ok_lz, n_lz + 1),
        (LZ4, "match_past_dn", bytes([0x4F]) + b"abcd" + b"\x01\x00\x20", 30),
        (SNAPPY, "offset_zero", _varint(12) + bytes([3 << 2]) + b"abcd" + bytes([2 | (7 << 2)]) + b"\x00\x00", 12),
        (SNAPPY, "offset_past_output", _varint(12) + bytes([3 << 2]) + b"abcd" + bytes([1 | (4 << 2), 5]), 12),
        (SNAPPY, "copy1_truncated", _varint(12) + bytes([3 << 2]) + b"abcd" + bytes([1 | (4 << 2)]), 12),
        (SNAPPY, "copy2_truncated", _varint(12) + bytes([3 << 2]) + b"abcd" + bytes([2 | (7 << 2), 4]), 12),
        (SNAPPY, "copy4_truncated", _varint(12) + bytes([3 << 2]) + b"abcd" + bytes([3 | (7 << 2), 4, 0, 0]), 12),
        (SNAPPY, "literal_length_bytes_truncated", _varint(300) + bytes([61 << 2, 0x2B]), 300),
        (SNAPPY, "literal_past_source", _varint(20) + bytes([19 << 2]) + b"x" * 10, 20),
        (SNAPPY, "copy_past_dn", _varint(12) + bytes([3 << 2]) + b"abcd" + bytes([2 | (15 << 2)]) + b"\x04\x00", 12),
        (SNAPPY, "length_too_small", ok_sn, n_sn - 1),
        (SNAPPY, "length_too_large", ok_sn, n_sn + 1),
        (SNAPPY, "varint_over_32_bits", b"\xff\xff\xff\xff\x1f" + lit20, 20),
        (SNAPPY, "varint_six_bytes", b"\x94\x80\x80\x80\x80\x00" + lit20, 20),
        (SNAPPY, "varint_truncated", b"\x80", 0),
        (SNAPPY, "empty_stream", b"", 0),
        # a 20-byte literal, then a literal of 0xFFFFFFF1 bytes: 32-bit sums of the length wrap below both limits
        (SNAPPY, "literal_length_wraps", _varint(40) + lit20 + bytes([0xFC, 0xF0, 0xFF, 0xFF, 0xFF]) + b"B" * 20, 40),
        (SNAPPY, "literal_length_2pow32", _varint(40) + lit20 + bytes([0xFC, 0xFF, 0xFF, 0xFF, 0xFF]) + b"B" * 20, 40),
        (STORED, "shorter_source", b"x" * 100, 101),
        (STORED, "longer_source", b"x" * 101, 100),
    ]
    return cases


# ---- child process: malformed and garbled streams ----------------------------------------------------------------------
def _child_malformed():
    """Every malformed case is refused (by both builds) with the canaries intact; pyarrow refuses them too."""
    errors = []
    for desc in (False, True):
        h = HostLz(desc)
        for codec, name, stream, dn in _malformed():
            for sph, dph in ((0, 0), (3, 9), (15, 1)):
                ok, _, intact = h(codec, stream, dn, sph, dph)
                if ok or not intact:
                    errors.append((codec, name, desc, sph, dph, ok, intact))
            if codec != STORED and reference(codec, stream, dn)[0]:
                errors.append((codec, name, "pyarrow accepts it"))
    return errors


def _garbled_sources(codec):
    rng = np.random.default_rng(79 + codec)
    words = [b"GET", b"POST", b"/api/v1/logs", b"200", b"404", b"upstream", b"timeout"]
    text = b"".join(b" ".join(words[j] for j in rng.integers(0, 7, 6)) + b"\n" for _ in range(600))
    hand = (lz4_streams() if codec == LZ4 else snappy_streams())["short_offsets" if codec == LZ4 else "copies"]
    return [(_PA[codec].compress(text, asbytes=True), text), hand]


def _lz4_zero_offset(stream):
    """Whether the sequences of an LZ4 block reach a match offset of 0.  The block format calls such a block corrupt
    and the decoder refuses it; pyarrow's LZ4 copies the bytes being written instead."""
    sp = 0
    while sp < len(stream):
        tok = stream[sp]
        sp += 1
        lit = tok >> 4
        while lit >= 15 and sp < len(stream):
            lit += stream[sp]
            sp += 1
            if stream[sp - 1] != 255:
                break
        sp += lit
        if sp + 2 > len(stream):
            return False
        if stream[sp] == 0 and stream[sp + 1] == 0:
            return True
        sp += 2
        if tok & 15 == 15:
            while sp < len(stream) and stream[sp] == 255:
                sp += 1
            sp += 1
    return False


def _child_fuzz(codec):
    """Bit flips: no write outside the destination, and agreement with pyarrow where it decodes exactly dn bytes.  The
    LZ4 decoder does not enforce the block's end rules (the last match 12 bytes before the end, the last 5 bytes
    literals) and refuses offset 0, so there only pyarrow's acceptance of an offset-free stream is checked."""
    rng = np.random.default_rng(83 + codec)
    hosts = (HostLz(False), HostLz(True))
    errors, refused, trials = [], 0, 0
    for stream, data in _garbled_sources(codec):
        for t in range(200):
            g = bytearray(stream)
            for _ in range(int(rng.integers(1, 4))):
                g[int(rng.integers(0, len(g)))] ^= 1 << int(rng.integers(0, 8))
            g = bytes(g)
            n = len(data) + (int(rng.integers(-3, 4)) if t % 5 == 0 else 0)
            n = max(n, 0)
            sph, dph = int(rng.integers(0, 16)), int(rng.integers(0, 16))
            ref_ok, ref_out = reference(codec, g, n)
            got = [h(codec, g, n, sph, dph) for h in hosts]
            trials += 1
            refused += not got[0][0]
            for desc, (ok, out, intact) in enumerate(got):
                if not intact:
                    errors.append(("canary", t, desc))
                if ok and ref_ok and out != ref_out:
                    errors.append(("bytes differ", t, desc))
                if ref_ok and not ok and not (codec == LZ4 and _lz4_zero_offset(g)):
                    errors.append(("refused what pyarrow decodes", t, desc))
                if codec == SNAPPY and ok and not ref_ok:
                    errors.append(("accepted what pyarrow refuses", t, desc))
            if got[0][:2] != got[1][:2]:
                errors.append(("lane orders differ", t))
    if refused < trials // 5:
        errors.append(("too few refusals", refused, trials))
    return errors


def _run_child(what):
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), what]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, f"child '{what}' exited with {r.returncode}\n{r.stdout[-4000:]}\n{r.stderr[-4000:]}"
    errors = json.loads(r.stdout.strip().splitlines()[-1])
    assert not errors, errors[:20]


# ---- CPU tests -----------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module", params=[False, True], ids=["lanes_up", "lanes_down"])
def host(request):
    return HostLz(request.param)


@pytest.mark.parametrize("codec", [LZ4, SNAPPY], ids=["lz4_raw", "snappy"])
def test_encoder_corpus(host, codec):
    """pyarrow's encodings of the zstd corpus decode to the same bytes, at a few source / destination phases."""
    for name, data in _inputs():
        comp = _PA[codec].compress(data, asbytes=True)
        for sph, dph in ((0, 0), (1, 0), (0, 7), (13, 6)):
            ok, out, intact = host(codec, comp, len(data), sph, dph)
            assert ok and intact and out == data, (name, sph, dph, len(data), len(comp))


@pytest.mark.parametrize("codec", [LZ4, SNAPPY], ids=["lz4_raw", "snappy"])
def test_hand_built_streams_at_every_phase(host, codec):
    streams = lz4_streams() if codec == LZ4 else snappy_streams()
    for name, (stream, data) in streams.items():
        ref_ok, ref_out = reference(codec, stream, len(data))
        assert ref_ok and ref_out == data, ("pyarrow does not decode the hand-built stream", name)
        for sph in range(16):
            for dph in range(16):
                ok, out, intact = host(codec, stream, len(data), sph, dph)
                assert ok and intact and out == data, (name, sph, dph)


def test_hand_built_streams_reach_every_form():
    """The encoder emits what the decoders' branches expect: length extensions ending in 0 and holding 255s, Snappy
    tags of all four kinds and literals with 0-4 length bytes."""
    lz = lz4_streams()
    assert b"\xff\x00" in lz["lit_ext"][0] and b"\xff\x01" in lz["lit_ext"][0]
    assert bytes([0xF1, 0x00]) in lz["lit_ext"][0]
    assert b"\x11\x00\x00" in lz["match_ext"][0] and b"\x11\x00\xff\x00" in lz["match_ext"][0]   # offset 17, extension 0 | 255 0
    sn = snappy_streams()["literal_lengths"][0] + snappy_streams()["copies"][0]
    for nb in (1, 2, 3, 4):
        assert bytes([(59 + nb) << 2]) in sn
    for kind in (1, 2, 3):
        assert any(b & 3 == kind for b in sn)


def test_stored_pages(host):
    rng = np.random.default_rng(89)
    for n in [0] + LIT_LENS:
        data = _rand(rng, n)
        for sph, dph in ((0, 0), (5, 0), (0, 11), (7, 3), (15, 15)):
            ok, out, intact = host(STORED, data, n, sph, dph)
            assert ok and intact and out == data, (n, sph, dph)


def test_malformed_streams_are_refused():
    _run_child("malformed")


@pytest.mark.parametrize("codec", [LZ4, SNAPPY], ids=["lz4_raw", "snappy"])
def test_garbled_streams(codec):
    _run_child(f"fuzz{codec}")


def test_heavy_pages_through_one_workspace():
    """ZSTD and GZIP pages decoded one after another through one workspace (the union a k_decompress_zstd warp
    reuses), alternating formats, so that every page starts from the tables and literals the previous one left."""
    import gzip
    lib = ctypes.CDLL(_so("libzstd_host.so"))
    P = ctypes.c_void_p
    lib.heavy_host_decode_run.argtypes = [ctypes.c_uint32, P, P, P, P, P, P, P, P]
    lib.heavy_host_decode_run.restype = ctypes.c_int
    pages = []
    for k, (name, data) in enumerate(_inputs()):
        pages.append((ZSTD, pa.Codec("zstd", compression_level=[1, 3, 19][k % 3]).compress(data, asbytes=True), data))
        pages.append((GZIP, gzip.compress(data, compresslevel=[1, 6, 9][k % 3]), data))
        pages.append((ZSTD, pa.Codec("zstd", compression_level=-5).compress(data, asbytes=True), data))
    codecs = np.array([p[0] for p in pages], np.uint32)
    src_len = np.array([len(p[1]) for p in pages], np.uint32)
    dst_len = np.array([len(p[2]) for p in pages], np.uint32)
    src_off = np.concatenate([[0], np.cumsum(src_len.astype(np.uint64))[:-1]]).astype(np.uint64)
    dst_off = np.concatenate([[0], np.cumsum(dst_len.astype(np.uint64) + 16)[:-1]]).astype(np.uint64)
    src = np.frombuffer(b"".join(p[1] for p in pages) + bytes(16), np.uint8).copy()
    dst = np.full(int(dst_off[-1]) + int(dst_len[-1]) + 16, FILL, np.uint8)
    ok = np.zeros(len(pages), np.int32)
    good = lib.heavy_host_decode_run(len(pages), codecs.ctypes.data, src.ctypes.data, src_off.ctypes.data, src_len.ctypes.data,
                                     dst.ctypes.data, dst_off.ctypes.data, dst_len.ctypes.data, ok.ctypes.data)
    assert good == len(pages) and ok.all(), ok
    for k, (codec, _, data) in enumerate(pages):
        o = int(dst_off[k])
        assert dst[o:o + len(data)].tobytes() == data, (k, codec)
        assert (dst[o + len(data):o + len(data) + 16] == FILL).all(), k


# ---- GPU tests: the kernels through launch_decompress ------------------------------------------------------------------
JOB = np.dtype([("src_off", "<u8"), ("dst_off", "<u8"), ("src_len", "<u4"), ("dst_len", "<u4"), ("codec", "<u4"), ("pad", "<u4")])


class DevImages:
    """Source and destination images for one launch of tools/libdecomp_dev.so.  Every job's payload sits at a chosen
    byte phase of the source; its destination either in a 16-byte aligned slot (a page) or at an odd offset (the values
    of a v2 page behind its levels), with FILL bytes between slots that must survive."""

    def __init__(self):
        self.src, self.jobs, self.want = bytearray(), [], []
        self.dst_size = 64

    def add(self, codec, stream, data, sphase=0, odd=False, dn=None):
        self.src += bytes((-len(self.src)) % 16 + sphase)
        so = len(self.src)
        self.src += stream
        dn = len(data) if dn is None else dn
        do = (self.dst_size + 15) // 16 * 16 + (7 if odd else 0)
        self.dst_size = do + dn + 48
        self.jobs.append((so, do, len(stream), dn, codec, 0))
        self.want.append(data)
        return len(self.jobs) - 1

    def run(self):
        lib = ctypes.CDLL(_so("libdecomp_dev.so"))
        P = ctypes.c_void_p
        lib.decomp_dev_run.argtypes = [P, ctypes.c_uint32, P, ctypes.c_uint64, P, ctypes.c_uint64, P]
        lib.decomp_dev_run.restype = ctypes.c_int
        jobs = np.array(self.jobs, JOB)
        src = np.frombuffer(bytes(self.src) or b"\x00", np.uint8).copy()
        dst = np.full(self.dst_size, FILL, np.uint8)
        flag = np.zeros(1, np.uint64)
        err = lib.decomp_dev_run(jobs.ctypes.data, len(jobs), src.ctypes.data, len(self.src), dst.ctypes.data, dst.size, flag.ctypes.data)
        assert err == 0, f"CUDA error {err}"
        return dst, int(flag[0])

    def check(self, dst, skip=()):
        """every job's bytes; FILL everywhere else (the jobs in `skip` must have written nothing)"""
        covered = np.zeros(dst.size, bool)
        for k, ((_, do, _, dn, codec, _), data) in enumerate(zip(self.jobs, self.want)):
            if k in skip:
                continue
            assert dst[do:do + dn].tobytes() == data, (k, codec, dn)
            covered[do:do + dn] = True
        assert (dst[~covered] == FILL).all(), np.flatnonzero((dst != FILL) & ~covered)[:20]


def _mixed_launch(bad=()):
    import gzip
    rng = np.random.default_rng(97)
    im = DevImages()
    k = 0
    for name, data in _inputs():
        for codec in (LZ4, SNAPPY, STORED):
            stream = data if codec == STORED else _PA[codec].compress(data, asbytes=True)
            im.add(codec, stream, data, sphase=k % 16, odd=k % 3 == 0)
            k += 1
    for codec, streams in ((LZ4, lz4_streams()), (SNAPPY, snappy_streams())):
        for name, (stream, data) in streams.items():
            for sph in range(16):
                im.add(codec, stream, data, sphase=sph, odd=sph % 2 == 1)
    # more ZSTD / GZIP pages than persistent warps (at most 2 CTAs of 4 warps per SM), so warps reuse their workspace
    # page after page, formats mixed
    n_heavy = 0
    while n_heavy < 1400:
        n = int(rng.integers(0, 3000))
        data = (b"%d " % rng.integers(0, 50)) * (n // 3) + _rand(rng, int(rng.integers(0, 64)))
        if n_heavy % 2:
            stream = gzip.compress(data, compresslevel=int(rng.integers(1, 10)))
            codec = GZIP
        else:
            stream = pa.Codec("zstd", compression_level=int(rng.choice([-5, 1, 3, 19]))).compress(data, asbytes=True)
            codec = ZSTD
        im.add(codec, stream, data, sphase=n_heavy % 16, odd=n_heavy % 5 == 0)
        n_heavy += 1
    bad_jobs = []
    for codec, stream, dn in bad:
        bad_jobs.append(im.add(codec, stream, b"", sphase=len(bad_jobs) % 16, dn=dn))
    return im, bad_jobs


@pytest.mark.gpu
def test_gpu_mixed_launch():
    im, _ = _mixed_launch()
    dst, flag = im.run()
    assert flag == 0
    im.check(dst)


@pytest.mark.gpu
def test_gpu_bad_jobs_among_good_ones():
    """Pages the decoders refuse before writing anything, among good ones: the flag is set, nothing of the bad jobs
    reaches the destination, and every good job still decodes exactly."""
    lit20 = bytes([19 << 2]) + b"A" * 20
    bad = [
        (STORED, b"x" * 100, 101),
        (STORED, b"x" * 101, 100),
        (SNAPPY, _varint(41) + lit20 + b"B" * 21, 40),                              # declared length differs
        (SNAPPY, b"\xff\xff\xff\xff\x1f" + lit20, 20),                             # varint over 32 bits
        (SNAPPY, _varint(40) + bytes([0xFC, 0xF0, 0xFF, 0xFF, 0xFF]) + b"B" * 40, 40),   # a first literal that wraps
        (SNAPPY, _varint(12) + bytes([2 | (7 << 2)]) + b"\x01\x00", 12),            # copy before any output
        (LZ4, bytes([0x00, 0x00, 0x00, 0x50]) + b"12345", 9),                       # offset 0, no literal before it
        (LZ4, bytes([0xF0]), 15),                                                   # truncated length extension
        (ZSTD, b"\x00" * 16, 10),                                                   # no frame magic
        (GZIP, b"\x00" * 32, 10),                                                   # no gzip magic
    ]
    im, bad_jobs = _mixed_launch(bad)
    dst, flag = im.run()
    assert flag == 1
    im.check(dst, skip=set(bad_jobs))
    for k in bad_jobs:
        _, do, _, dn, _, _ = im.jobs[k]
        assert (dst[do:do + dn] == FILL).all(), k


if __name__ == "__main__":
    what = sys.argv[1]
    errs = _child_malformed() if what == "malformed" else _child_fuzz(int(what[4:]))
    print(json.dumps([[str(x) for x in e] for e in errs]))
