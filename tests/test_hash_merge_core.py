"""The merge of a hashed GROUP BY's rank tables under PQ_QUERY_ALLREDUCE, on the CPU: the host build of hash_merge.cuh
(tools/libhash_merge_host.so, built with -ffp-contract=off) against a Python fold in rank order.

Each run gathers N <= 8 ranks' blocks as the all-gather lays them out: 1 + cells planes of E_max words per rank (wide
ids, then the cell planes), the first E_r records listed, the rest padding.  A rank's wide ids are distinct (one hash
table cell per group), listed in ascending or in random order.  The merge must give:
- the groups in ascending wide id, each once;
- count, COUNT and non-null planes and Int64 SUM as wrapping sums;
- Float64 SUM / AVG as f64 adds in rank order (((r0 + r1) + r2) ...), bit for bit;
- MIN / MAX as signed min / max of the cell encoding (totalOrder for Float64), +-0 and NaN payloads included."""
import ctypes as C
import os
import struct
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "tools", "libhash_merge_host.so")
ADD, F64, MIN, MAX = 0, 1, 2, 3
M64 = (1 << 64) - 1


@pytest.fixture(scope="module")
def lib(built):
    if not os.path.exists(LIB):
        subprocess.check_call(["make", "-C", ROOT, os.path.relpath(LIB, ROOT)])
    h = C.CDLL(LIB)
    h.hm_merge.restype = C.c_uint32
    h.hm_merge.argtypes = [C.c_uint32, C.c_uint64, C.c_uint32, C.c_uint32, C.c_char_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    h.hm_combine_host.restype = C.c_uint64
    h.hm_combine_host.argtypes = [C.c_uint64, C.c_uint64, C.c_uint32]
    return h


def f64_bits(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def bits_f64(b):
    return struct.unpack("<d", struct.pack("<Q", b))[0]


def total_order(b):
    """The signed cell encoding of a Float64 for MIN / MAX (IEEE totalOrder), as unsigned 64 bits."""
    mag = b & ((1 << 63) - 1)
    return ((-mag - 1) & M64) if b >> 63 else mag


def s64(u):
    return u - (1 << 64) if u >> 63 else u


F64_POOL = [0.0, -0.0, 1.5, -2.25, 1e300, -1e300, 3.0e-310, float("inf"), float("-inf"), 0.1, 1 / 3]
NAN_BITS = [0x7FF8000000000001, 0xFFF8000000000002, 0x7FF0000000000F00, 0xFFF0000000000007]


def cell_value(rng, how, nan_ok):
    if how == ADD:
        return int(rng.integers(0, 1 << 64, dtype=np.uint64))
    if how == F64:
        if nan_ok and rng.random() < 0.05:
            return NAN_BITS[rng.integers(len(NAN_BITS))]
        if rng.random() < 0.5:
            return f64_bits(F64_POOL[rng.integers(len(F64_POOL))])
        return f64_bits(float(rng.normal() * 10.0 ** rng.integers(-5, 6)))
    # MIN / MAX: totalOrder codes of Float64 values (NaN payloads and +-0 included) or plain Int64
    if rng.random() < 0.5:
        b = NAN_BITS[rng.integers(len(NAN_BITS))] if rng.random() < 0.2 else f64_bits(F64_POOL[rng.integers(len(F64_POOL))])
        return total_order(b)
    return int(rng.integers(-(1 << 63), (1 << 63) - 1)) & M64


def python_fold(blocks, listed, hows):
    """{wide id: [cell words]} folded in rank order."""
    out = {}
    for r, (ids, planes) in enumerate(blocks):
        for j in range(listed[r]):
            w = ids[j]
            cur = out.get(w)
            vals = [planes[c][j] for c in range(len(hows))]
            if cur is None:
                out[w] = vals
                continue
            for c, how in enumerate(hows):
                a, b = cur[c], vals[c]
                if how == ADD:
                    cur[c] = (a + b) & M64
                elif how == F64:
                    cur[c] = f64_bits(bits_f64(a) + bits_f64(b))
                elif how == MIN:
                    cur[c] = b if s64(b) < s64(a) else a
                else:
                    cur[c] = b if s64(b) > s64(a) else a
    return out


def run_merge(lib, blocks, listed, e_max, n_acc, acc_init, hows):
    nr, cells = len(blocks), len(hows)
    recv = np.zeros((nr, 1 + cells, max(e_max, 1)), np.uint64)
    for r, (ids, planes) in enumerate(blocks):
        recv[r, 0, :e_max] = ids
        for c in range(cells):
            recv[r, 1 + c, :e_max] = planes[c]
    recv = np.ascontiguousarray(recv[:, :, :e_max]) if e_max else np.zeros(1, np.uint64)
    lst = np.array(listed, np.uint64)
    cap = max(int(lst.sum()), 1)
    acc = np.zeros(cells * cap, np.uint64)
    wide = np.zeros(cap, np.uint64)
    g = lib.hm_merge(nr, e_max, cells, n_acc, bytes(acc_init), recv.ctypes.data, lst.ctypes.data, acc.ctypes.data, wide.ctypes.data)
    return g, wide[:g].tolist(), acc.reshape(cells, cap)[:, :g]


def check(lib, rng, nr, e_max, n_acc, n_nn, sorted_ids, key_space, nan_ok=True):
    acc_init = [int(x) for x in rng.integers(0, 4, n_acc)]
    hows = [ADD] + acc_init + [ADD] * n_nn
    cells = len(hows)
    # wide ids drawn from a small pool so that ranks share groups; one rank may list nothing
    pool = rng.choice(key_space, size=min(key_space, max(1, int(e_max * 1.5))), replace=False).astype(np.uint64)
    blocks, listed = [], []
    for r in range(nr):
        e = int(rng.integers(0, e_max + 1)) if r else e_max   # rank 0 lists E_max records
        if rng.random() < 0.15:
            e = 0 if r else e
        ids = rng.choice(pool, size=min(e, len(pool)), replace=False)
        e = len(ids)
        if sorted_ids:
            ids = np.sort(ids)
        pad = rng.integers(0, 1 << 64, e_max - e, dtype=np.uint64)   # padding: never read
        planes = [[cell_value(rng, how, nan_ok) for _ in range(e)] + [int(x) for x in rng.integers(0, 1 << 64, e_max - e, dtype=np.uint64)]
                  for how in hows]
        blocks.append((np.concatenate([ids.astype(np.uint64), pad]).tolist(), planes))
        listed.append(e)
    e_max = max(listed) if listed else 0
    blocks = [(ids[:e_max] + [0] * (e_max - len(ids[:e_max])), [p[:e_max] for p in planes]) for ids, planes in blocks]
    want = python_fold(blocks, listed, hows)
    g, wide, acc = run_merge(lib, blocks, listed, e_max, n_acc, acc_init, hows)
    what = (nr, e_max, n_acc, n_nn, sorted_ids, listed)
    assert g == len(want), what
    assert wide == sorted(want), what          # ascending wide id, each group once
    for gi, w in enumerate(wide):
        for c, how in enumerate(hows):
            got, exp = int(acc[c, gi]), want[w][c]
            if how == F64 and bits_f64(exp) != bits_f64(exp):
                assert bits_f64(got) != bits_f64(got), (what, w, c)   # NaN of arithmetic: its payload is not specified
            else:
                assert got == exp, (what, w, c, hex(got), hex(exp))


@pytest.mark.parametrize("seed", range(40))
def test_merge_random_runs(lib, seed):
    rng = np.random.default_rng(20261018 + seed)
    nr = int(rng.integers(1, 9))
    check(lib, rng, nr, int(rng.integers(0, 300)), int(rng.integers(0, 9)), int(rng.integers(0, 4)), bool(seed % 2),
          int(rng.choice([1 << 27, 1 << 40, 1 << 62])))


def test_merge_f64_sum_in_rank_order(lib):
    """1e16 + 1 + 1 + ... differs from the sum of the small terms first: the fold keeps rank order, bit for bit."""
    nr = 8
    vals = [1e16] + [1.0] * 7
    blocks = [([5], [[1], [f64_bits(v)]]) for v in vals]
    g, wide, acc = run_merge(lib, blocks, [1] * nr, 1, 1, [F64], [ADD, F64])
    exp = 0.0
    for k, v in enumerate(vals):
        exp = v if k == 0 else exp + v
    assert g == 1 and wide == [5]
    assert int(acc[1, 0]) == f64_bits(exp) and exp == 1e16   # each +1 rounds away: ((1e16 + 1) + 1) ...
    assert int(acc[0, 0]) == nr


def test_merge_min_max_total_order(lib):
    """Signed min / max of totalOrder codes: -NaN < -inf < -0 < +0 < +inf < +NaN, payloads ordered."""
    order = [0xFFF8000000000002, f64_bits(float("-inf")), f64_bits(-1.0), f64_bits(-0.0), f64_bits(0.0), f64_bits(2.0),
             f64_bits(float("inf")), 0x7FF0000000000F00, 0x7FF8000000000001]
    codes = [total_order(b) for b in order]
    assert [s64(c) for c in codes] == sorted(s64(c) for c in codes)
    perm = [4, 0, 8, 3, 6, 1, 7, 5]   # rank r holds order[perm[r]]
    blocks = [([9], [[1], [codes[p]], [codes[p]]]) for p in perm]
    g, _, acc = run_merge(lib, blocks, [1] * len(perm), 1, 2, [MIN, MAX], [ADD, MIN, MAX])
    assert g == 1
    assert int(acc[1, 0]) == codes[min(perm)] and int(acc[2, 0]) == codes[max(perm)]


def test_merge_wrapping_sums(lib):
    big = (1 << 63) - 5
    blocks = [([1, 2], [[3, 1], [big, M64]]), ([2, 1], [[2, 2], [10, big]])]
    g, wide, acc = run_merge(lib, blocks, [2, 2], 2, 1, [ADD], [ADD, ADD])
    assert g == 2 and wide == [1, 2]
    assert acc[:, 0].tolist() == [5, (2 * big) & M64]
    assert acc[:, 1].tolist() == [3, 9]


def test_merge_nothing_listed(lib):
    g, wide, _ = run_merge(lib, [([], [[]]) for _ in range(3)], [0, 0, 0], 0, 0, [], [ADD])
    assert g == 0 and wide == []


def test_combine(lib):
    assert lib.hm_combine_host(M64, 2, ADD) == 1
    assert lib.hm_combine_host(f64_bits(0.1), f64_bits(0.2), F64) == f64_bits(0.1 + 0.2)
    assert lib.hm_combine_host(f64_bits(-0.0), f64_bits(-0.0), F64) == f64_bits(-0.0)
    assert lib.hm_combine_host(5, M64, MIN) == M64          # -1 < 5
    assert lib.hm_combine_host(5, M64, MAX) == 5
