"""Brute-force neighbour tables of the sparse convolutions (layers.SparseConv / SparseConvTranspose): every (output,
input) pair in numpy float32, in the order of oracle_sparse_conv (oracle/ops_ref.c): product rounded, + offset,
+ kernel_size / 2, floor.  One input per (output, kernel cell), the lowest id; the count of non-empty cells."""
from fractions import Fraction

import numpy as np


def brute_table(inp, out, v, offset, ks, transpose=False, chunk=128):
    """int64 [M, kx*ky*kz] table (shadow id N) and int64 [M] count of non-empty cells."""
    inp, out = np.asarray(inp, np.float32).reshape(-1, 3), np.asarray(out, np.float32).reshape(-1, 3)
    n, m = len(inp), len(out)
    ks = np.asarray(ks, np.int64).reshape(3)
    kc = int(ks.prod())
    inv_v = np.float32(1) / np.float32(v)
    off = np.asarray(offset, np.float32).reshape(3)
    half = (np.float32(0.5) * ks.astype(np.float32)).astype(np.float32)
    table = np.full((m, kc), n, np.int64)
    for o0 in range(0, m, chunk):
        o = out[o0:o0 + chunk]
        d = (o[:, None, :] - inp[None]) if transpose else (inp[None] - o[:, None, :])
        r = ((d * inv_v).astype(np.float32) + off).astype(np.float32)
        c = np.floor((r + half).astype(np.float32)).astype(np.int64)
        ok = ((c >= 0) & (c < ks)).all(2)
        oo, ii = np.nonzero(ok)                          # row-major: ascending input id inside an output
        cell = (c[oo, ii, 0] * ks[1] + c[oo, ii, 1]) * ks[2] + c[oo, ii, 2]
        key, first = np.unique(oo * kc + cell, return_index=True)
        table[o0 + key // kc, key % kc] = ii[first]
    return table, (table < n).sum(1)


def contract64(feat, table, kernel):
    """float64 [M, Cout] = sum over the cells c of kernel[c]^T feat[table[:, c]]; the shadow id reads zeros."""
    f = np.concatenate([np.asarray(feat, np.float64), np.zeros((1, feat.shape[1]))])
    t = np.minimum(table, len(feat))
    w = np.asarray(kernel, np.float64).reshape(table.shape[1], feat.shape[1], -1)
    return sum(f[t[:, c]] @ w[c] for c in range(table.shape[1]))


def round_f32(x):
    """A Fraction rounded to the nearest float32, ties to even (no detour through a float64 rounding)."""
    y = np.float32(float(x))
    best = None
    for c in (np.nextafter(y, np.float32(-np.inf)), y, np.nextafter(y, np.float32(np.inf))):
        e = abs(Fraction(float(c)) - x)
        if best is None or e < best[0] or (e == best[0] and int(c.view(np.int32)) % 2 == 0):
            best = (e, c)
    return best[1]


def face_points(v, off, ks, transpose, count, seed):
    """(input, output) float32 coordinate pairs on one axis whose cell differs between the unfused predicate
    floor(round(round(d * inv_v) + off) + ks / 2) and one that fuses the product into the offset add, each confirmed
    in exact rational arithmetic.  Candidates are inputs a few ulps around the cell faces out + (k - off - ks/2) v."""
    rng = np.random.default_rng(seed)
    inv_v = np.float32(1) / np.float32(v)
    off, half = np.float32(off), np.float32(0.5 * ks)
    out = (rng.random(200000) * 40 - 20).astype(np.float32)
    k = rng.integers(0, ks + 1, 200000)
    face = (out.astype(np.float64) + (k - float(off) - 0.5 * ks) * float(v) * (-1 if transpose else 1))
    inp = np.float32(face)
    inp = np.nextafter(inp, np.float32(np.inf) * np.sign(rng.random(200000) - 0.5).astype(np.float32))
    pairs = []
    for step in range(4):
        d = (out - inp) if transpose else (inp - out)
        unfused = np.floor(((d * inv_v).astype(np.float32) + off).astype(np.float32) + half)
        approx = np.floor((np.float32(d.astype(np.float64) * float(inv_v) + float(off))) + half)
        for i in np.nonzero(unfused != approx)[0]:
            exact = round_f32(Fraction(float(d[i])) * Fraction(float(inv_v)) + Fraction(float(off)))
            if np.floor(np.float32(exact + half)) != unfused[i]:
                pairs.append((inp[i], out[i]))
        inp = np.nextafter(inp, np.float32(np.inf) * (1 if step % 2 else -1))
        if len(pairs) >= count:
            break
    return pairs[:count]
