"""Every non-table instance of gemm_tc_kernel (csrc/gemm_tc.cu) against float64, crossed with the modes and epilogue
paths it can reach: rows (o3dml_linear_tc), the 3x3 convolution at stride 1 and 2, the 3x3x3 convolution and the
transposed convolution with its pixel-shuffle epilogue.  gemm_tc_launch picks the instance at run time from the shape
and the SM count, so each case derives its shape from the SM count through gemm_tc_support.route, and the profiler trace
must show that exact instance, launched once.  The output starts as NaN, so an element the kernel skips fails the
comparison, and every element outside the written region must still be NaN afterwards."""
import math

import pytest
import torch
import torch.nn.functional as F

from open3d_ml_b200 import _lib as L

from conftest import rel_err
from gemm_tc_support import (GATHER, LITE, MATRIX_INSTANCES, PLAIN, ROWS, TABLE_INSTANCES, conv3x3_tiles,
                             conv3x3x3_tiles, inst_name, launched_instances, n_pad, route, traced,
                             traced_instance)
from test_gpu_dense import DENSE_TOL, _gathered

SLOPE = 0.1
POOL = 300           # rows of a gathered source


def long_k_tol(k):
    """The bound on rel_err for a product of K = k.  Each fold of the accumulator (every 128 channels) adds one fp32
    rounding of the running sum, and those roundings add up like a random walk, so the error grows as sqrt(K) for K
    beyond the 2304 (= 9 x 256) of the longest convolution DENSE_TOL was measured on.  On an H100 80GB HBM3 (700 W power
    limit) the largest rel_err was 1.17e-6 at K = 4096 (bound 9.3e-6) and 1.11e-6 at K = 8192 (bound 1.3e-5); over the
    whole matrix it was 1.49e-6, so the error did not grow with K over that range."""
    return DENSE_TOL * max(1.0, math.sqrt(k / 2304))


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def at(v, S):
    """A case dimension: a number, or a function of the SM count."""
    return v(S) if callable(v) else v


def tiles_over(f):
    """The fewest 128-row tiles t with t * f > sms(): the least grid that fills the SMs more than once."""
    return lambda S: S // f + 1


def gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def randn(*shape, seed):
    return torch.randn(*shape, generator=gen(seed), device="cuda")


def rows_with_tail(t):
    return (t - 1) * ROWS + 37


def round4(c):
    return (c + 3) // 4 * 4


def epilogue_ref(y, s, t, res, act, axis):
    """float64 act(y * s + t + res), s and t per channel along `axis`."""
    shape = [1] * y.dim()
    shape[axis] = -1
    if s is not None:
        y = y * s.double().view(shape)
    if t is not None:
        y = y + t.double().view(shape)
    if res is not None:
        y = y + res
    if act == "relu":
        return y.clamp_min(0)
    if act == "leaky":
        return torch.where(y >= 0, y, y * SLOPE)
    return y


def affine(cout, ep, seed):
    """ep 'ss': scale and shift, 't': shift only, '-': neither."""
    s = randn(cout, seed=seed).abs() + 0.5 if ep == "ss" else None
    t = randn(cout, seed=seed + 1) if ep in ("ss", "t") else None
    return s, t


def nan_out(rows, cout, out):
    """A NaN-filled output: 'rows' [rows, cout], 'slice4' a 16-byte aligned channel slice with out_ld % 4 == 0 of a wider
    buffer, 'slice1' a slice at column 1 with out_ld % 4 != 0.  -> (buffer, view, out_ld, first column)."""
    if out == "rows":
        buf = torch.full((rows, cout), float("nan"), device="cuda")
        return buf, buf, cout, 0
    width, c0 = (round4(cout) + 8, 4) if out == "slice4" else (cout + 7 if (cout + 7) % 4 else cout + 6, 1)
    buf = torch.full((rows, width), float("nan"), device="cuda")
    return buf, buf[:, c0:c0 + cout], width, c0


def untouched(buf, c0, cout):
    """Every element of the buffer outside the channel slice [c0, c0 + cout) of its last axis is still NaN."""
    return bool(buf[..., :c0].isnan().all()) and bool(buf[..., c0 + cout:].isnan().all())


class Built:
    """One prepared call: run() enqueues it, got() is its output as float64 in the layout of ref, affected the outputs
    (rows / pixels / voxels, broadcast over channels) that read a poisoned input, inside() the outside-is-NaN check."""

    def __init__(self, run, got, ref, inside, k, buf, affected=None):
        self.run, self.got, self.ref, self.inside, self.k, self.buf, self.affected = (run, got, ref, inside, k, buf,
                                                                                      affected)


def _poison(x, picks):
    """NaN, +Inf and -Inf at three row positions of x (one channel each); -> the poisoned copy and a 0/1 row mask."""
    mask = torch.zeros(x.shape[0], device="cuda")
    x = x.clone()
    for p, v in zip(picks, (float("nan"), float("inf"), float("-inf"))):
        x[p, (7 * p) % x.shape[1]] = v
        mask[p] = 1
    return x, mask


class Rows:
    """o3dml_linear_tc.  srcs: (channels, kind) per source, kind 'id' (the output row itself), 'g32' / 'g64' (global
    int32 / int64 ids, column 0 of an [n, 2] matrix, -1 and == rows read zeros), 'batch' (int64 ids relative to two batch
    items; ids == and past src_rows_per_batch read zeros).  res: None, 'al' (16-byte rows), 'ld' (res_ld % 4 != 0) or
    'off' (the pointer one float past 16-byte alignment).  out: 'rows', 'slice4', 'slice1' or 'nchw' (two planes)."""

    def __init__(self, n, srcs, cout, ep="ss", act="leaky", res=None, out="rows"):
        self.n, self.srcs, self.cout, self.ep, self.act, self.res, self.out = n, srcs, cout, ep, act, res, out

    def target(self, S):
        n = at(self.n, S)
        k = sum(c for c, _ in self.srcs)
        return route(-(-n // ROWS), self.cout, k, S, gather=any(kind != "id" for _, kind in self.srcs))

    def build(self, S, seed, mag=1.0, poison=False):
        n = at(self.n, S)
        cout, keep, srcs, cols = self.cout, [], [], []
        affected = torch.zeros(n, dtype=torch.bool, device="cuda")
        for j, (ch, kind) in enumerate(self.srcs):
            kw = {}
            if kind == "id":
                data = randn(n, ch, seed=seed + j) * mag
            else:
                data = randn(POOL, ch, seed=seed + j) * mag
                if kind in ("g32", "g64"):
                    idx = torch.randint(-1, POOL + 1, (n, 2), generator=gen(seed + 10 + j), device="cuda")
                    idx[:2, 0] = torch.tensor([-1, POOL], device="cuda")[:min(n, 2)]
                    kw = dict(index=idx.to(torch.int32 if kind == "g32" else torch.int64), index_ld=2)
                else:
                    spb = POOL // 2
                    idx = torch.randint(0, spb + 2, (n,), generator=gen(seed + 10 + j), device="cuda")
                    idx[:2] = torch.tensor([spb, spb + 1], device="cuda")[:min(n, 2)]
                    kw = dict(index=idx, out_rows_per_batch=(n + 1) // 2, src_rows_per_batch=spb)
            if poison and j == 0:        # three rows of the first source that some output row reads
                rid = _gathered(torch.arange(1, data.shape[0] + 1, device="cuda").double()[:, None], n, **kw)[:, 0]
                read = rid[rid > 0].unique()
                picks = sorted({int(read[i]) - 1 for i in (0, len(read) // 2, -1)})
                clean = data
                data, mask = _poison(data, picks)
                affected = _gathered(mask[:, None], n, **kw)[:, 0] > 0
                cols.append(_gathered(clean, n, **kw))
            else:
                cols.append(_gathered(data, n, **kw))
            keep.append((data, kw))
            srcs.append(L.make_src(data, **kw))
        k = sum(c for c, _ in self.srcs)
        w = randn(k, cout, seed=seed + 20) / k ** 0.5
        pw = L.pack_linear(w)
        s, t = affine(cout, self.ep, seed + 21)
        r, rld, rref = None, 0, None
        if self.res is not None:
            if self.res == "off":
                rld = round4(cout)
                r = randn(n * rld + 1, seed=seed + 23)[1:].view(n, rld)[:, :cout]
            else:
                rld = round4(cout) + 4 if self.res == "al" else (cout + 1 if (cout + 1) % 4 else cout + 2)
                r = randn(n, rld, seed=seed + 23)[:, :cout]
            rref = r.double()
        plane = 0
        if self.out == "nchw":
            assert n % 2 == 0
            plane = n // 2
            buf = torch.full((2, cout, plane), float("nan"), device="cuda")
            o, ld, c0 = buf, cout, 0
            got = lambda: buf.permute(0, 2, 1).reshape(n, cout).double()          # noqa: E731
            inside = lambda: True                                                  # noqa: E731
        else:
            buf, o, ld, c0 = nan_out(n, cout, self.out)
            got = lambda: o.double()                                               # noqa: E731
            inside = lambda: untouched(buf, c0, cout)                              # noqa: E731
        ref = epilogue_ref(torch.cat(cols, 1) @ w.double(), s, t, rref, self.act, 1)
        arr = (L.Src * len(srcs))(*srcs)
        keep += [arr, pw, s, t, r]

        def run(_keep=keep):
            return L.lib().o3dml_linear_tc(n, arr, len(srcs), L.ptr(pw.img), pw.k_pad, pw.n_pad, L.ptr(s), L.ptr(t),
                                           L.ptr(r), rld, L.act_code(self.act), SLOPE, L.ptr(o), ld, cout, plane,
                                           L.stream())
        return Built(run, got, ref, inside, k, buf, affected[:, None])


class Conv3x3:
    """_lib.conv3x3 on a PackedWeight: NHWC [B, H, W, C] -> [B, OH, OW, cout], padding 1."""

    def __init__(self, B, H, W, C, cout, stride, ep="ss", act="relu"):
        self.B, self.H, self.W, self.C, self.cout, self.stride, self.ep, self.act = B, H, W, C, cout, stride, ep, act

    def target(self, S):
        B = at(self.B, S)
        return route(B * conv3x3_tiles(self.H, self.W, self.stride), self.cout, 9 * self.C, S, rows_mode=False)

    def build(self, S, seed, mag=1.0, poison=False):
        B = at(self.B, S)
        H, W, C, co, st = self.H, self.W, self.C, self.cout, self.stride
        x = randn(B, H, W, C, seed=seed) * mag
        w = randn(co, C, 3, 3, seed=seed + 1) / (9 * C) ** 0.5
        s, t = affine(co, self.ep, seed + 2)
        OH, OW = (H - 1) // st + 1, (W - 1) // st + 1
        affected = torch.zeros(B, OH, OW, 1, dtype=torch.bool, device="cuda")
        clean = x
        if poison:
            flat, mask = _poison(x.view(-1, C), [0, (B * H * W) // 2 + W // 2, B * H * W - 1])
            x = flat.view(B, H, W, C)
            hit = F.conv2d(mask.view(B, 1, H, W).double(), torch.ones(1, 1, 3, 3, dtype=torch.float64, device="cuda"),
                           None, st, 1)
            affected = (hit > 0).permute(0, 2, 3, 1)
        out = torch.full((B, OH, OW, co), float("nan"), device="cuda")
        pw = L.pack_linear(w.permute(2, 3, 1, 0).reshape(9 * C, co).contiguous())
        ref = F.conv2d(clean.permute(0, 3, 1, 2).double(), w.double(), None, st, 1)
        ref = epilogue_ref(ref, s, t, None, self.act, 1).permute(0, 2, 3, 1)

        def run():
            L.conv3x3(x, pw, out, s, t, st, act=self.act, slope=SLOPE)
        return Built(run, lambda: out.double(), ref, lambda: True, 9 * C, out, affected)


class Conv3x3x3:
    """_lib.conv3x3x3: channels-last grids [B, X, Y, Z, C] -> [B, X, Y, Z, cout], padding 1."""

    def __init__(self, B, dims, C, cout, ep="ss", act="relu"):
        self.B, self.dims, self.C, self.cout, self.ep, self.act = B, dims, C, cout, ep, act

    def target(self, S):
        B = at(self.B, S)
        return route(B * conv3x3x3_tiles(*self.dims), self.cout, 27 * self.C, S, rows_mode=False)

    def build(self, S, seed, mag=1.0, poison=False):
        B = at(self.B, S)
        (X, Y, Z), C, co = self.dims, self.C, self.cout
        x = randn(B, X, Y, Z, C, seed=seed) * mag
        w = randn(co, C, 3, 3, 3, seed=seed + 1) / (27 * C) ** 0.5
        s, t = affine(co, self.ep, seed + 2)
        affected = torch.zeros(B, X, Y, Z, 1, dtype=torch.bool, device="cuda")
        clean = x
        if poison:
            nv = B * X * Y * Z
            flat, mask = _poison(x.view(-1, C), [0, nv // 2 + (Y * Z) // 2 + Z // 2, nv - 1])
            x = flat.view(B, X, Y, Z, C)
            hit = F.conv3d(mask.view(B, 1, X, Y, Z).double(),
                           torch.ones(1, 1, 3, 3, 3, dtype=torch.float64, device="cuda"), None, 1, 1)
            affected = (hit > 0).permute(0, 2, 3, 4, 1)
        out = torch.full((B, X, Y, Z, co), float("nan"), device="cuda")
        pw = L.pack_linear(w.permute(2, 3, 4, 1, 0).reshape(27 * C, co).contiguous())
        ref = F.conv3d(clean.permute(0, 4, 1, 2, 3).double(), w.double(), None, 1, 1)
        ref = epilogue_ref(ref, s, t, None, self.act, 1).permute(0, 2, 3, 4, 1)

        def run():
            L.conv3x3x3(x, pw, out, s, t, act=self.act, slope=SLOPE)
        return Built(run, lambda: out.double(), ref, lambda: True, 27 * C, out, affected)


class Deconv:
    """_lib.deconv (kernel == stride) on a PackedWeight: a rows-mode product over the input pixels, C -> stride^2 cout
    columns, pixel-shuffled into [B, H s, W s, cout], which is the whole NaN buffer ('rows') or a channel slice of it."""

    def __init__(self, B, H, W, C, cout, stride, ep="ss", act="relu", out="slice4"):
        self.B, self.H, self.W, self.C, self.cout, self.stride = B, H, W, C, cout, stride
        self.ep, self.act, self.out = ep, act, out

    def target(self, S):
        B, H, W = (at(v, S) for v in (self.B, self.H, self.W))
        return route(-(-B * H * W // ROWS), self.stride ** 2 * self.cout, self.C, S)

    def build(self, S, seed, mag=1.0, poison=False):
        B, H, W = (at(v, S) for v in (self.B, self.H, self.W))
        C, co, st = self.C, self.cout, self.stride
        x = randn(B, H, W, C, seed=seed) * mag
        w = randn(C, co, st, st, seed=seed + 1) / C ** 0.5
        s, t = affine(co, self.ep, seed + 2)
        affected = torch.zeros(B, H * st, W * st, 1, dtype=torch.bool, device="cuda")
        clean = x
        if poison:
            flat, mask = _poison(x.view(-1, C), [0, (B * H * W) // 2 + W // 2, B * H * W - 1])
            x = flat.view(B, H, W, C)
            affected = mask.view(B, H, W).repeat_interleave(st, 1).repeat_interleave(st, 2)[..., None] > 0
        buf, _, _, c0 = nan_out(1, co, self.out)
        buf = torch.full((B, H * st, W * st, buf.shape[1]), float("nan"), device="cuda")
        o = buf[..., c0:c0 + co]
        pw = L.pack_linear(w.permute(0, 2, 3, 1).reshape(C, st * st * co).contiguous())
        s_rep = None if s is None else s.repeat(st * st)
        t_rep = None if t is None else t.repeat(st * st)
        ref = F.conv_transpose2d(clean.permute(0, 3, 1, 2).double(), w.double(), None, st)
        ref = epilogue_ref(ref, s, t, None, self.act, 1).permute(0, 2, 3, 1)

        def run(_keep=(s_rep, t_rep)):
            L.deconv(x, pw, o, s_rep, t_rep, st, act=self.act, slope=SLOPE)
        return Built(run, lambda: o.double(), ref, lambda: untouched(buf, c0, co), C, buf, affected)


def per_tile(f):
    """Rows that make exactly tiles_over(f) 128-row tiles, the last one ragged."""
    return lambda S: rows_with_tail(tiles_over(f)(S))


def lite_rows(S):
    return (S + 2) * ROWS


# id -> (the instance the case targets, the case).  Column counts 1 .. 257 cover the 32 / 64 / 128-multiple padding of
# the weight image and ragged column tiles; K 4 .. 8192 covers sub-slice products, the 16-slice LITE limit, one slice
# past it, and many accumulator folds and wraps of the stage ring.
CASES = {
    # ---- <32, GATHER>
    "g32_three_srcs_ragged": (GATHER[32], Rows(1000, [(32, "id"), (32, "g32"), (20, "id")], 31, "ss", "leaky", "ld",
                                                "slice1")),
    "g32_int64_nchw": (GATHER[32], Rows(130, [(64, "g64")], 32, "t", "relu", None, "nchw")),
    "g32_batch_one_row": (GATHER[32], Rows(1, [(28, "batch")], 3, "ss", "none")),
    # ---- <64, GATHER>
    "g64_batch_res_off": (GATHER[64], Rows(127, [(32, "batch"), (4, "id")], 63, "ss", "leaky", "off")),
    "g64_k516_nchw": (GATHER[64], Rows(600, [(32, "id"), (32, "g64"), (452, "id")], 65, "ss", "relu", "al", "nchw")),
    "g64_slice4": (GATHER[64], Rows(128, [(32, "g32")], 33, "-", "none", None, "slice4")),
    # ---- <128, GATHER>: the RandLA-Net decoder (skip rows and batch-relative coarse rows)
    "g128_decoder": (GATHER[128], Rows(per_tile(2), [(32, "id"), (64, "batch")], 128, "ss", "leaky", "ld")),
    "g128_long_k": (GATHER[128], Rows(per_tile(4), [(2048, "g32"), (2052, "id")], 129, "t", "none", "off",
                                      "slice1")),
    "g128_nchw": (GATHER[128], Rows(lambda S: 2 * (S // 12 + 1) * ROWS, [(32, "g64"), (32, "id"), (12, "id")], 257,
                                    "ss", "relu", "al", "nchw")),
    # ---- <32, LITE>
    "l32_k512": (LITE[32], Rows(lambda S: rows_with_tail(S + 2), [(512, "id")], 32, "ss", "leaky", "al")),
    "l32_k4_cout1": (LITE[32], Rows(lite_rows, [(4, "id")], 1, "t", "none", "ld", "slice1")),
    "l32_nchw_head": (LITE[32], Rows(lite_rows, [(384, "id")], 31, "ss", "none", "off", "nchw")),
    # ---- <64, LITE>
    "l64_k28_slice4": (LITE[64], Rows(lambda S: (S + 1) * ROWS + 1, [(28, "id")], 64, "-", "relu", None, "slice4")),
    "l64_three_srcs": (LITE[64], Rows(per_tile(2), [(32, "id"), (32, "id"), (20, "id")], 65, "ss", "leaky", "ld")),
    "l64_cout257_nchw": (LITE[64], Rows(lambda S: 2 * (S // 12 + 1) * ROWS, [(512, "id")], 257, "t", "none", "al",
                                        "nchw")),
    "l64_cout127_res_off": (LITE[64], Rows(per_tile(2), [(32, "id")], 127, "ss", "relu", "off", "slice1")),
    # ---- <32> (no gather, no LITE)
    "p32_one_row": (PLAIN[32], Rows(1, [(4, "id")], 31, "ss", "leaky")),
    "p32_127_rows": (PLAIN[32], Rows(127, [(28, "id")], 3, "t", "relu", "al", "slice1")),
    "p32_128_rows_nchw": (PLAIN[32], Rows(128, [(32, "id")], 32, "-", "none", "off", "nchw")),
    "p32_k516": (PLAIN[32], Rows(129, [(516, "id")], 1, "ss", "leaky", "ld", "slice4")),
    "p32_long_k": (PLAIN[32], Rows(rows_with_tail(7), [(4096, "id")], 17, "ss", "none")),
    "p32_many_tiles": (PLAIN[32], Rows(lambda S: (S + 1) * ROWS, [(512, "id"), (32, "id"), (4, "id")], 32, "ss",
                                       "leaky")),
    # ---- <64>
    "p64_one_row": (PLAIN[64], Rows(1, [(4, "id")], 63, "t", "none", None, "slice4")),
    "p64_k512_nchw": (PLAIN[64], Rows(130, [(512, "id")], 33, "ss", "relu", "ld", "nchw")),
    "p64_cout65": (PLAIN[64], Rows(600, [(516, "id")], 65, "ss", "leaky", "al")),
    "p64_cout129": (PLAIN[64], Rows(1000, [(28, "id")], 129, "ss", "none", "off", "slice1")),
    "p64_cout257": (PLAIN[64], Rows(128, [(32, "id")], 257, "t", "leaky")),
    "p64_k8192": (PLAIN[64], Rows(rows_with_tail(3), [(8192, "id")], 64, "ss", "none")),
    # ---- <128>
    "p128_k516": (PLAIN[128], Rows(per_tile(2), [(516, "id")], 127, "ss", "leaky", "ld")),
    "p128_long_k": (PLAIN[128], Rows(per_tile(4), [(4096, "id")], 129, "t", "none", "al", "slice4")),
    "p128_cout257_nchw": (PLAIN[128], Rows(lambda S: 2 * (S // 12 + 1) * ROWS, [(1024, "id")], 257, "ss", "relu", "off",
                                           "nchw")),
    "p128_three_srcs": (PLAIN[128], Rows(per_tile(2), [(256, "id"), (256, "id"), (36, "id")], 65, "ss", "none", None,
                                         "slice1")),
    # ---- the 3x3 convolution (never LITE, never gathered)
    "conv_s1_p32": (PLAIN[32], Conv3x3(2, 9, 7, 32, 31, 1, "ss", "leaky")),
    "conv_s2_p64": (PLAIN[64], Conv3x3(1, 20, 16, 64, 64, 2, "t", "relu")),
    "conv_s2_p64_cout129": (PLAIN[64], Conv3x3(1, 13, 13, 128, 129, 2, "-", "none")),
    "conv_s1_p128": (PLAIN[128], Conv3x3(lambda S: -(-(S // 2 + 1) // conv3x3_tiles(62, 54, 1)), 62, 54, 64, 128, 1,
                                         "ss", "relu")),
    "conv_s2_p128": (PLAIN[128], Conv3x3(lambda S: -(-(S // 4 + 1) // conv3x3_tiles(62, 54, 2)), 62, 54, 32, 256, 2,
                                         "ss", "leaky")),
    # ---- the 3x3x3 convolution
    "conv3d_p32": (PLAIN[32], Conv3x3x3(2, (9, 7, 5), 32, 31, "ss", "leaky")),
    "conv3d_p64": (PLAIN[64], Conv3x3x3(1, (16, 16, 16), 64, 64, "t", "none")),
    "conv3d_p128": (PLAIN[128], Conv3x3x3(lambda S: -(-(S // 2 + 1) // conv3x3x3_tiles(24, 24, 24)), (24, 24, 24), 32,
                                          128, "ss", "relu")),
    # ---- the transposed convolution: staged (cout % 4 == 0) and element-wise pixel shuffles
    "deconv_s4_l64": (LITE[64], Deconv(1, lambda S: (S // 32) * ROWS // 27 + 1, 27, 128, 128, 4, "ss", "relu",
                                       "slice4")),
    "deconv_s2_l32_cout6": (LITE[32], Deconv(1, 128, lambda S: S + 2, 64, 6, 2, "t", "leaky", "slice1")),
    "deconv_s1_l64_unaligned": (LITE[64], Deconv(1, lambda S: S + 1, 129, 64, 64, 1, "ss", "none", "slice1")),
    "deconv_s4_l64_cout6": (LITE[64], Deconv(1, lambda S: (S // 2) * ROWS // 95 + 1, 95, 32, 6, 4, "ss", "leaky",
                                             "slice4")),
    "deconv_s2_p64_cout10": (PLAIN[64], Deconv(2, 6, 5, 64, 10, 2, "ss", "relu", "slice4")),
    "deconv_s4_p64_cout12": (PLAIN[64], Deconv(1, 9, 7, 96, 12, 4, "t", "leaky", "slice1")),
    "deconv_s2_p32_cout5": (PLAIN[32], Deconv(2, 1, 5, 32, 5, 2, "-", "none", "rows")),
    "deconv_s2_p128": (PLAIN[128], Deconv(1, lambda S: (S // 4) * ROWS // 72 + 1, 72, 544, 64, 2, "ss", "relu",
                                          "slice4")),
    "deconv_s1_p128_cout130": (PLAIN[128], Deconv(1, lambda S: (S // 4) * ROWS // 67 + 1, 67, 516, 130, 1, "-", "none",
                                                  "rows")),
}


def test_every_instance_has_cases():
    """The instances gemm_tc.cu launches are the matrix's and the table mode's, one GT_INSTANCES entry each: adding or
    removing an instance without its cases fails here."""
    assert launched_instances() == sorted(MATRIX_INSTANCES + TABLE_INSTANCES)
    assert sorted({tgt for tgt, _ in CASES.values()}) == MATRIX_INSTANCES


def test_route_matches_the_documented_rule():
    """The Python copy of gemm_tc_launch's rule on the H100 SXM's 132 SMs and the H100 PCIe's 114, at the boundaries
    the cases lean on."""
    for S in (114, 132):
        assert route(S, 32, 512, S) == PLAIN[32] and route(S + 1, 32, 512, S) == LITE[32]
        assert route(S + 1, 32, 516, S) == PLAIN[32]
        assert route(S // 2 + 1, 128, 512, S) == LITE[64] and route(S // 2, 128, 512, S) == PLAIN[64]
        assert route(S // 2 + 1, 128, 516, S) == PLAIN[128] and route(S // 2, 128, 516, S) == PLAIN[64]
        assert route(S // 2 + 1, 128, 64, S, gather=True) == GATHER[128]
        assert route(S // 2, 128, 64, S, gather=True) == GATHER[64]
        assert route(S // 2 + 1, 128, 64, S, rows_mode=False) == PLAIN[128]
        assert route(10 * S, 20, 64, S, gather=True) == GATHER[32]
    assert n_pad(1) == 32 and n_pad(33) == 64 and n_pad(65) == 128 and n_pad(129) == 256 and n_pad(257) == 384


def run_traced(tgt, built):
    """Runs the call under the profiler: one launch, of instance tgt."""
    counted, names = traced(built.run)
    assert counted == 1 and traced_instance(names) == [tgt], (inst_name(tgt), counted, names)


def check_values(built, tol):
    got, ref = built.got(), built.ref
    assert not bool(got.isnan().any()), "an output element was not written"
    err = rel_err(got, ref)
    assert err < tol, (err, tol)
    assert built.inside(), "an element outside the output region was written"
    return err


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_instance_matrix_vs_float64(case):
    """The case reaches its instance, matches float64 within the bound for its K, and a second run is bit-equal."""
    tgt, spec = CASES[case]
    S = sms()
    assert spec.target(S) == tgt, "case %s no longer reaches %s on %d SMs" % (case, inst_name(tgt), S)
    b = spec.build(S, seed=list(CASES).index(case))
    run_traced(tgt, b)
    err = check_values(b, long_k_tol(b.k))
    first = b.buf.clone()
    b.run()
    assert torch.equal(first.view(torch.int32), b.buf.view(torch.int32)), "two runs differ"
    print("%s %s K=%d rel_err=%.3g" % (case, inst_name(tgt), b.k, err))


MAGNITUDE_CASES = ["l64_k28_slice4", "l32_k512", "g128_decoder", "conv_s1_p128", "conv_s2_p64"]


@pytest.mark.gpu
@pytest.mark.parametrize("mag", [1e-20, 1e20])
@pytest.mark.parametrize("case", MAGNITUDE_CASES)
def test_magnitude_independent(case, mag):
    """The TF32 split keeps fp32's exponent: inputs scaled by 1e-20 or 1e20, no shift or residual to hide them, hold the
    same relative bound."""
    tgt, spec = CASES[case]
    spec = type(spec)(**{**vars(spec), "ep": "-", "act": "none", **({"res": None} if hasattr(spec, "res") else {})})
    S = sms()
    b = spec.build(S, seed=7, mag=mag)
    run_traced(tgt, b)
    check_values(b, long_k_tol(b.k))


CONTAINMENT_CASES = ["g32_three_srcs_ragged", "g64_batch_res_off", "g128_decoder", "l32_k4_cout1", "l64_three_srcs",
                     "p32_127_rows", "p64_cout129", "p128_k516", "conv_s1_p32", "conv_s2_p64", "conv_s1_p128",
                     "conv3d_p64", "deconv_s4_l64", "deconv_s2_l32_cout6"]


@pytest.mark.gpu
@pytest.mark.parametrize("case", CONTAINMENT_CASES)
def test_non_finite_input_stays_contained(case):
    """NaN, +Inf and -Inf in three input rows / pixels / voxels make exactly the outputs that read them non-finite (in
    every channel; +Inf may come out as NaN, since the split's lo = Inf - Inf), and leave every other output finite and
    within the bound.  relu is replaced by leaky here: fmaxf(NaN, 0) is 0, so relu hides a NaN."""
    tgt, spec = CASES[case]
    if spec.act == "relu":
        spec = type(spec)(**{**vars(spec), "act": "leaky"})
    S = sms()
    b = spec.build(S, seed=11, poison=True)
    run_traced(tgt, b)
    got = b.got()
    bad = ~torch.isfinite(got)
    expect = b.affected.expand_as(got)
    assert int(expect.any(-1).sum()) >= 1
    assert torch.equal(bad, expect), (int(bad.sum()), int(expect.sum()))
    keep = ~expect
    assert rel_err(got[keep], b.ref[keep]) < long_k_tol(b.k)
    assert b.inside()


@pytest.mark.gpu
@pytest.mark.parametrize("n,cin,cout", [(30000, 64, 64), (20011, 96, 128), (40000, 128, 32)])
def test_linear_plain_lite_rows_run_lite(n, cin, cout, monkeypatch):
    """The rows of test_gpu_dense.py::test_linear_plain that its comment calls LITE run a LITE instance, the one route
    names, under that module's routing.  The trace is taken here, not there: with profiling sessions opened in
    test_gpu_dense.py, every session after test_gpu_detect.py in the same process came back without activity records."""
    monkeypatch.setattr(L, "USE_ROW_MLP", False)
    x, w = randn(n, cin, seed=1), randn(cin, cout, seed=2) / cin ** 0.5
    out = torch.full((n, cout), float("nan"), device="cuda")
    pw = L.pack_linear(w)
    tgt = route(-(-n // ROWS), cout, cin, sms())
    assert tgt[2]
    counted, names = traced(lambda: L.linear([L.make_src(x)], pw, out, act=None))
    assert counted == 1 and traced_instance(names) == [tgt], (inst_name(tgt), names)
    assert rel_err(out, x.double() @ w.double()) < DENSE_TOL
