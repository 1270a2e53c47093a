"""A small Parquet writer for tests: Thrift compact page headers and footers, and stream encoders that follow an
explicit plan, so that a test can write the stream shapes the format allows but pyarrow's writer never emits.

Every encoder has a plain reference decoder next to it, written from the format specification
(https://github.com/apache/parquet-format: Encodings.md, parquet.thrift).  Nothing here is tuned for speed."""
from __future__ import annotations

import struct
from dataclasses import dataclass, field

import numpy as np
import pyarrow as pa

# parquet.thrift enums
PT_BOOLEAN, PT_INT32, PT_INT64, PT_DOUBLE, PT_BYTE_ARRAY = 0, 1, 2, 5, 6
PLAIN, PLAIN_DICTIONARY, RLE, DELTA_BINARY_PACKED, DELTA_LENGTH_BYTE_ARRAY, DELTA_BYTE_ARRAY, RLE_DICTIONARY = 0, 2, 3, 5, 6, 7, 8
DATA_PAGE, DICTIONARY_PAGE, DATA_PAGE_V2 = 0, 2, 3
CODECS = {"NONE": 0, "SNAPPY": 1, "GZIP": 2, "ZSTD": 6, "LZ4_RAW": 7}
MASK64 = (1 << 64) - 1

# column kinds: physical type, Arrow type
KINDS = {"i64": (PT_INT64, pa.int64()), "f64": (PT_DOUBLE, pa.float64()), "str": (PT_BYTE_ARRAY, pa.string()),
         "bool": (PT_BOOLEAN, pa.bool_()), "ts": (PT_INT64, pa.timestamp("ms")), "date": (PT_INT32, pa.date32())}


# ---- Thrift compact protocol -----------------------------------------------------------------------------------------
T_TRUE, T_FALSE, T_I32, T_I64, T_BINARY, T_LIST, T_STRUCT = 1, 2, 5, 6, 8, 9, 12


def uleb(v: int) -> bytes:
    assert v >= 0
    out = bytearray()
    while True:
        b = v & 0x7F
        v >>= 7
        if v:
            out.append(b | 0x80)
        else:
            out.append(b)
            return bytes(out)


def zigzag(v: int) -> int:
    return ((v << 1) ^ (v >> 63)) & MASK64


def unzigzag(z: int) -> int:
    return (z >> 1) ^ -(z & 1)


def _tval(t, v) -> bytes:
    if t in (T_I32, T_I64):
        return uleb(zigzag(v))
    if t == T_BINARY:
        v = v.encode() if isinstance(v, str) else v
        return uleb(len(v)) + v
    if t == T_STRUCT:
        return v
    if t == T_LIST:
        et, items = v
        head = bytes([(len(items) << 4) | et]) if len(items) < 15 else bytes([0xF0 | et]) + uleb(len(items))
        return head + b"".join(_tval(et, x) for x in items)
    raise AssertionError(t)


def tstruct(*fields) -> bytes:
    """fields: (id, type, value); value None leaves the field out; T_TRUE stands for a bool field of value `value`."""
    out, last = bytearray(), 0
    for fid, t, v in fields:
        if v is None:
            continue
        if t == T_TRUE:
            t, v = (T_TRUE if v else T_FALSE), None
        d = fid - last
        out += bytes([(d << 4) | t]) if 0 < d <= 15 else bytes([t]) + uleb(zigzag(fid))
        if v is not None:
            out += _tval(t, v)
        last = fid
    out.append(0)
    return bytes(out)


# ---- RLE / bit-packed hybrid ----------------------------------------------------------------------------------------
def pack_bits(values, bw: int) -> bytes:
    acc = 0
    for i, v in enumerate(values):
        acc |= int(v) << (i * bw)
    return acc.to_bytes((len(values) * bw + 7) // 8, "little")


def encode_hybrid(runs, bw: int) -> bytes:
    """runs: ("rle", value, count) or ("bp", values, groups[, pad]).  A bit-packed run holds groups * 8 slots; the slots
    after `values` hold `pad` (0 by default), as a writer may leave them."""
    out = bytearray()
    for r in runs:
        if r[0] == "rle":
            _, v, n = r
            out += uleb(n << 1) + int(v).to_bytes((bw + 7) // 8, "little")
        else:
            vals, groups = list(r[1]), r[2]
            pad = r[3] if len(r) > 3 else 0
            assert len(vals) <= groups * 8
            out += uleb((groups << 1) | 1) + pack_bits(vals + [pad] * (groups * 8 - len(vals)), bw)
    return bytes(out)


def decode_hybrid(buf: bytes, bw: int, n: int, pos: int = 0):
    """-> (values, runs as (kind, count) with the slots each run holds, end position).  Reference decoder."""
    vals, runs = [], []
    vbytes = (bw + 7) // 8
    while len(vals) < n:
        h, shift = 0, 0
        while True:
            b = buf[pos]
            pos += 1
            h |= (b & 0x7F) << shift
            shift += 7
            if not b & 0x80:
                break
        if h & 1:
            groups = h >> 1
            acc = int.from_bytes(buf[pos:pos + groups * bw], "little")
            pos += groups * bw
            m = (1 << bw) - 1
            vals += [(acc >> (i * bw)) & m for i in range(groups * 8)]
            runs.append(("bp", groups * 8))
        else:
            v = int.from_bytes(buf[pos:pos + vbytes], "little")
            pos += vbytes
            vals += [v] * (h >> 1)
            runs.append(("rle", h >> 1))
    return vals[:n], runs, pos


def runs_for(values, bw, rng, max_bp_groups=40, rle_min=1):
    """A mixed plan over `values`: RLE runs (of 1 too) where values repeat or by chance, bit-packed runs elsewhere."""
    runs, i, n = [], 0, len(values)
    while i < n:
        j = i
        while j < n and values[j] == values[i]:
            j += 1
        if j - i >= rle_min and (j - i >= 8 or rng.random() < 0.3):
            runs.append(("rle", values[i], j - i))
            i = j
        else:
            g = int(rng.integers(1, max_bp_groups + 1))
            take = min(g * 8, n - i)
            runs.append(("bp", list(values[i:i + take]), (take + 7) // 8))
            i += take
    return runs


def def_runs(valid, rng, style="mixed"):
    """Definition levels (bit width 1) of a page: 'bp' writes bit-packed groups only, 'mixed' RLE where levels repeat."""
    lv = [int(x) for x in valid]
    if style == "bp":
        return [("bp", lv, (len(lv) + 7) // 8)] if lv else []
    return runs_for(lv, 1, rng, rle_min=9)


# ---- DELTA_BINARY_PACKED ---------------------------------------------------------------------------------------------
@dataclass
class DeltaPlan:
    """A stream's geometry: `block` values per block in `minis` miniblocks; widths(b, m) is miniblock m's width in
    block b, min_delta(b) the block's min delta; `junk` the bytes written as the unused widths of the last block."""
    block: int = 128
    minis: int = 4
    widths: object = None
    min_delta: object = None
    junk: int = 0


def delta_stream(n: int, plan: DeltaPlan, rng, bits=64, first=None):
    """Values drawn to fit the plan exactly (every delta = min delta + a random offset of the miniblock's width) and
    the stream that holds them.  bits=32: an INT32 stream (arithmetic wraps at 32 bits).  -> (values, bytes)"""
    mod = 1 << bits
    sgn = lambda x: x - mod if x >= mod // 2 else x  # noqa: E731
    vpm = plan.block // plan.minis
    first = int(rng.integers(-(1 << (bits - 2)), 1 << (bits - 2))) if first is None else first
    vals = [first]
    out = bytearray(uleb(plan.block) + uleb(plan.minis) + uleb(n) + uleb(zigzag(first) & (mod - 1 if bits == 32 else MASK64)))
    b, cur = 0, first % mod
    while len(vals) < n:
        md = plan.min_delta(b) if plan.min_delta else int(rng.integers(-1000, 1000))
        ws = [plan.widths(b, m) if plan.widths else int(rng.integers(0, 12)) for m in range(plan.minis)]
        left = n - len(vals)
        used = min(plan.minis, -(-left // vpm))
        ws = ws[:used] + [plan.junk] * (plan.minis - used) if used < plan.minis else ws
        out += uleb(zigzag(md) if bits == 64 else zigzag(md) & 0xFFFFFFFF)
        out += bytes(ws)
        for m in range(used):
            w = ws[m]
            offs = [int(x) for x in rng.integers(0, 1 << w, vpm, dtype=np.uint64, endpoint=False)] if 0 < w < 64 else \
                [int(x) for x in rng.integers(0, 1 << 63, vpm, dtype=np.uint64)] if w == 64 else [0] * vpm
            if w == 64:
                offs = [o | (int(rng.integers(0, 2)) << 63) for o in offs]
            out += pack_bits(offs, w)
            for o in offs[:n - len(vals)]:
                cur = (cur + md + o) % mod
                vals.append(sgn(cur))
        b += 1
    return vals, bytes(out)


def decode_delta(buf: bytes, pos: int = 0, bits=64):
    """-> (values, geometry (block, minis), per-block widths, end position).  Reference decoder: the last miniblock
    with values is stored in full, later ones not at all (their widths are not read)."""
    def rd():
        nonlocal pos
        v, s = 0, 0
        while True:
            c = buf[pos]
            pos += 1
            v |= (c & 0x7F) << s
            s += 7
            if not c & 0x80:
                return v
    mod = 1 << bits
    block, minis, total, first = rd(), rd(), rd(), unzigzag(rd())
    vpm = block // minis
    vals, cur, widths = ([first] if total else []), first % mod, []
    while len(vals) < total:
        md = unzigzag(rd())
        ws = list(buf[pos:pos + minis])
        pos += minis
        used = []
        for w in ws:
            if len(vals) >= total:
                break
            used.append(w)
            acc = int.from_bytes(buf[pos:pos + vpm * w // 8], "little")
            pos += vpm * w // 8
            for i in range(vpm):
                if len(vals) >= total:
                    break
                cur = (cur + md + ((acc >> (i * w)) & ((1 << w) - 1))) % mod
                vals.append(cur - mod if cur >= mod // 2 else cur)
        widths.append(used)
    return vals, (block, minis), widths, pos


def delta_encode_values(vals, plan: DeltaPlan, bits=64) -> bytes:
    """A stream of given values under the plan's geometry (widths as the values need them; junk past the last)."""
    mod = 1 << bits
    n = len(vals)
    vpm = plan.block // plan.minis
    out = bytearray(uleb(plan.block) + uleb(plan.minis) + uleb(n) + uleb(zigzag(vals[0] if n else 0)))
    deltas = [((vals[i] - vals[i - 1] + mod // 2) % mod) - mod // 2 for i in range(1, n)]
    for b0 in range(0, len(deltas), plan.block):
        blk = deltas[b0:b0 + plan.block]
        md = min(blk)
        out += uleb(zigzag(md))
        used = -(-len(blk) // vpm)
        bodies, ws = bytearray(), []
        for m in range(used):
            offs = [(d - md) % mod for d in blk[m * vpm:(m + 1) * vpm]]
            w = max(offs).bit_length()
            ws.append(w)
            bodies += pack_bits(offs + [0] * (vpm - len(offs)), w)
        out += bytes(ws + [plan.junk] * (plan.minis - used)) + bodies
    return bytes(out)


# ---- byte arrays --------------------------------------------------------------------------------------------------------
def encode_dlba(strs, plan: DeltaPlan) -> bytes:
    return delta_encode_values([len(s) for s in strs], plan, 32) + b"".join(strs)


def encode_dba(strs, plan: DeltaPlan) -> bytes:
    pre, prev = [], b""
    for s in strs:
        k = 0
        while k < min(len(s), len(prev)) and s[k] == prev[k]:
            k += 1
        pre.append(k)
        prev = s
    return (delta_encode_values(pre, plan, 32) + delta_encode_values([len(s) - k for s, k in zip(strs, pre)], plan, 32)
            + b"".join(s[k:] for s, k in zip(strs, pre)))


def decode_dlba(buf: bytes, pos: int = 0):
    lens, _, _, pos = decode_delta(buf, pos, 32)
    out = []
    for n in lens:
        out.append(bytes(buf[pos:pos + n]))
        pos += n
    return out


def decode_dba(buf: bytes, pos: int = 0):
    pre, _, _, pos = decode_delta(buf, pos, 32)
    suf, _, _, pos = decode_delta(buf, pos, 32)
    out, prev = [], b""
    for p, s in zip(pre, suf):
        prev = prev[:p] + bytes(buf[pos:pos + s])
        pos += s
        out.append(prev)
    return out


# ---- PLAIN ------------------------------------------------------------------------------------------------------------
def encode_plain(kind: str, vals) -> bytes:
    if kind in ("i64", "ts"):
        return struct.pack(f"<{len(vals)}q", *vals)
    if kind == "f64":   # values are IEEE bit patterns (NaN payloads and -0.0 survive)
        return struct.pack(f"<{len(vals)}Q", *vals)
    if kind == "date":
        return struct.pack(f"<{len(vals)}i", *vals)
    if kind == "bool":
        return pack_bits([int(v) for v in vals], 1)
    if kind == "str":
        return b"".join(struct.pack("<I", len(s)) + s for s in vals)
    raise AssertionError(kind)


def decode_plain(kind: str, buf: bytes, n: int, pos: int = 0):
    if kind in ("i64", "ts"):
        return list(struct.unpack_from(f"<{n}q", buf, pos))
    if kind == "f64":
        return list(struct.unpack_from(f"<{n}Q", buf, pos))
    if kind == "date":
        return list(struct.unpack_from(f"<{n}i", buf, pos))
    if kind == "bool":
        acc = int.from_bytes(buf[pos:pos + (n + 7) // 8], "little")
        return [bool((acc >> i) & 1) for i in range(n)]
    out = []
    for _ in range(n):
        k = struct.unpack_from("<I", buf, pos)[0]
        out.append(bytes(buf[pos + 4:pos + 4 + k]))
        pos += 4 + k
    return out


# ---- pages, chunks, files ----------------------------------------------------------------------------------------------
@dataclass
class Page:
    """One data page.  `values`: the page's row values (None = NULL).  `enc`: the value encoding; `body`: the encoded
    non-null values (for dictionary pages the indices' hybrid stream, `bw` its width).  v2: levels outside the codec;
    `compressed` is the header's is_compressed."""
    values: list
    enc: int
    body: bytes
    v2: bool = False
    compressed: bool = True
    bw: int | None = None
    defs: list | None = None          # explicit definition-level runs (bit width 1); None: derived from the NULLs
    def_style: str = "mixed"
    plan: object = None               # what the test promises about the stream (read back from the file on the CPU)


@dataclass
class Chunk:
    pages: list
    dictionary: list | None = None    # dictionary entries (source values)
    dict_enc: int = PLAIN
    stats: bool = False
    dict_offset_field: bool = True    # False: dictionary page at data_page_offset, dictionary_page_offset unset
    gap: int = 0                      # bytes written before the chunk


@dataclass
class Column:
    name: str
    kind: str
    required: bool = False
    chunks: list = field(default_factory=list)   # one per row group

    def values(self):
        return [v for c in self.chunks for p in c.pages for v in p.values]


def _stat_bytes(kind, v):
    if kind in ("i64", "ts"):
        return struct.pack("<q", v)
    if kind == "f64":
        return struct.pack("<Q", v)
    if kind == "date":
        return struct.pack("<i", v)
    if kind == "bool":
        return bytes([int(v)])
    return v


def _f64_key(b):
    return struct.unpack("<d", struct.pack("<Q", b))[0]


def _stats(col: Column, vals):
    nn = [v for v in vals if v is not None]
    nulls = len(vals) - len(nn)
    if not nn:
        return tstruct((3, T_I64, nulls))
    if col.kind == "f64":
        fl = [x for x in nn if _f64_key(x) == _f64_key(x)]   # NaNs are left out of min / max
        if not fl:
            return tstruct((3, T_I64, nulls))
        lo, hi = min(fl, key=_f64_key), max(fl, key=_f64_key)
    else:
        lo, hi = min(nn), max(nn)
    return tstruct((3, T_I64, nulls), (5, T_BINARY, _stat_bytes(col.kind, hi)), (6, T_BINARY, _stat_bytes(col.kind, lo)))


def _compress(codec: str, b: bytes) -> bytes:
    return b if codec == "NONE" else pa.compress(b, codec=codec.lower(), asbytes=True)


def _page_bytes(col: Column, pg: Page, codec: str):
    """-> (header + payload as stored, header + payload uncompressed)"""
    valid = [v is not None for v in pg.values]
    levels = b""
    if not col.required:
        runs = pg.defs if pg.defs is not None else def_runs(valid, np.random.default_rng(len(valid)), pg.def_style)
        levels = encode_hybrid(runs, 1)
    body = pg.body
    n = len(pg.values)
    if pg.enc in (PLAIN_DICTIONARY, RLE_DICTIONARY):
        body = (bytes([pg.bw]) + body) if (pg.bw is not None) else body
    if pg.enc == RLE:
        body = struct.pack("<I", len(body)) + body
    if not pg.v2:
        raw = (struct.pack("<I", len(levels)) + levels if not col.required else b"") + body
        comp = _compress(codec, raw)
        h = tstruct((1, T_I32, DATA_PAGE), (2, T_I32, len(raw)), (3, T_I32, len(comp)),
                    (5, T_STRUCT, tstruct((1, T_I32, n), (2, T_I32, pg.enc), (3, T_I32, RLE), (4, T_I32, RLE))))
        return h + comp, len(h) + len(raw)
    vb = _compress(codec, body) if pg.compressed else body
    h = tstruct((1, T_I32, DATA_PAGE_V2), (2, T_I32, len(levels) + len(body)), (3, T_I32, len(levels) + len(vb)),
                (8, T_STRUCT, tstruct((1, T_I32, n), (2, T_I32, n - sum(valid)), (3, T_I32, n), (4, T_I32, pg.enc),
                                      (5, T_I32, len(levels)), (6, T_I32, 0), (7, T_TRUE, pg.compressed))))
    return h + levels + vb, len(h) + len(levels) + len(body)


def write_file(path: str, cols: list, codec: str = "NONE"):
    """Every column has one chunk per row group; the row groups' row counts come from the first column."""
    n_rg = len(cols[0].chunks)
    out = bytearray(b"PAR1")
    rgs = []
    for g in range(n_rg):
        ccs, rows = [], None
        for col in cols:
            ch = col.chunks[g]
            nrows = sum(len(p.values) for p in ch.pages)
            assert rows is None or nrows == rows, (col.name, nrows, rows)
            rows = nrows
            out += b"\0" * ch.gap
            start = len(out)
            dict_off = None
            uncomp = 0                        # total_uncompressed_size: headers + uncompressed payloads
            encs = {RLE}
            if ch.dictionary is not None:
                dict_off = len(out)
                raw = encode_plain(col.kind, ch.dictionary)
                comp = _compress(codec, raw)
                h = tstruct((1, T_I32, DICTIONARY_PAGE), (2, T_I32, len(raw)), (3, T_I32, len(comp)),
                            (7, T_STRUCT, tstruct((1, T_I32, len(ch.dictionary)), (2, T_I32, ch.dict_enc))))
                out += h + comp
                uncomp += len(h) + len(raw)
                encs.add(ch.dict_enc)
            data_off = len(out) if (ch.dictionary is None or ch.dict_offset_field) else start
            for pg in ch.pages:
                b, n_raw = _page_bytes(col, pg, codec)
                out += b
                uncomp += n_raw
                encs.add(pg.enc)
            size = len(out) - start
            vals = [v for p in ch.pages for v in p.values]
            meta = tstruct((1, T_I32, KINDS[col.kind][0]), (2, T_LIST, (T_I32, sorted(encs))), (3, T_LIST, (T_BINARY, [col.name])),
                           (4, T_I32, CODECS[codec]), (5, T_I64, len(vals)), (6, T_I64, uncomp), (7, T_I64, size),
                           (9, T_I64, data_off), (11, T_I64, dict_off if ch.dict_offset_field else None),
                           (12, T_STRUCT, _stats(col, vals) if ch.stats else None))
            ccs.append(tstruct((2, T_I64, start), (3, T_STRUCT, meta)))
        rgs.append(tstruct((1, T_LIST, (T_STRUCT, ccs)), (2, T_I64, 0), (3, T_I64, rows)))
    schema = [tstruct((4, T_BINARY, "schema"), (5, T_I32, len(cols)))]
    for col in cols:
        logical = {"str": tstruct((1, T_STRUCT, tstruct())), "date": tstruct((6, T_STRUCT, tstruct())),
                   "ts": tstruct((8, T_STRUCT, tstruct((1, T_TRUE, False), (2, T_STRUCT, tstruct((1, T_STRUCT, tstruct()))))))}.get(col.kind)
        conv = {"str": 0, "date": 6, "ts": 9}.get(col.kind)
        schema.append(tstruct((1, T_I32, KINDS[col.kind][0]), (3, T_I32, 0 if col.required else 1), (4, T_BINARY, col.name),
                              (6, T_I32, conv), (10, T_STRUCT, logical)))
    nrows = sum(sum(len(p.values) for p in cols[0].chunks[g].pages) for g in range(n_rg))
    meta = tstruct((1, T_I32, 1), (2, T_LIST, (T_STRUCT, schema)), (3, T_I64, nrows), (4, T_LIST, (T_STRUCT, rgs)),
                   (6, T_BINARY, "parquet_forge"))
    out += meta + struct.pack("<I", len(meta)) + b"PAR1"
    with open(path, "wb") as f:
        f.write(out)


# ---- page constructors ------------------------------------------------------------------------------------------------
def dict_page(values, dictionary, runs, bw, **kw) -> Page:
    """A dictionary-index page: `values` are the row values (None = NULL); `runs` the hybrid plan over the indices of the
    non-null ones."""
    return Page(values=values, enc=kw.pop("enc", RLE_DICTIONARY), body=encode_hybrid(runs, bw), bw=bw,
                plan=kw.pop("plan", ("hybrid", bw, [(r[0], r[2] if r[0] == "rle" else r[2] * 8) for r in runs])), **kw)


def plain_page(kind, values, **kw) -> Page:
    return Page(values=values, enc=PLAIN, body=encode_plain(kind, [v for v in values if v is not None]), **kw)


def to_arrow(col: Column) -> pa.Array:
    vals = col.values()
    t = KINDS[col.kind][1]
    if col.kind == "f64":
        bits = np.array([0 if v is None else v for v in vals], np.uint64)
        return pa.Array.from_buffers(pa.float64(), len(vals), [pa.array([v is not None for v in vals]).buffers()[1],
                                                               pa.py_buffer(bits.view(np.float64).tobytes())],
                                     null_count=sum(v is None for v in vals))
    if col.kind == "str":
        return pa.array(vals, pa.binary()).cast(pa.string())
    if col.kind == "ts":
        return pa.array(vals, pa.int64()).cast(t)
    if col.kind == "date":
        return pa.array(vals, pa.int32()).cast(t)
    return pa.array(vals, t)
