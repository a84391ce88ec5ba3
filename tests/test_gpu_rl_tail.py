"""The fused RandLA-Net tail (rl_tail.cu: last decoder SharedMLP on [skip | nearest_interpolation(x)] + the fc1 stack)
through its C ABI, against a float64 restatement of the four layers: class counts, partial and multi-wave tiles,
int32 / int64 and batch-relative / global interpolation indices, indices that select no coarse row, strided rows,
magnitudes, output bounds, schedule invariance and argument validation."""
import pytest
import torch

from open3d_ml_b200 import _lib as L
from conftest import elem_err, rel_err

pytestmark = pytest.mark.gpu

NAN = float("nan")
PAD = 128           # sentinel rows behind every output
SLOPE = 0.2


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def make_weights(classes, seed, bn=True):
    """wd [64, 32], w0 [32, 64], w1 [64, 32], w3 [32, classes] ([in, out]) and the host scale / shift [4][64]."""
    g = torch.Generator().manual_seed(seed)
    shapes = [(64, 32), (32, 64), (64, 32), (32, classes)]
    ws = [torch.randn(k, n, generator=g) / k ** 0.5 for k, n in shapes]
    scale, shift = torch.ones(4, 64), torch.zeros(4, 64)
    if bn:
        for li, (_, n) in enumerate(shapes):
            scale[li, :n] = torch.rand(n, generator=g) + 0.5
            shift[li, :n] = torch.randn(n, generator=g) * 0.1
    return ws, scale.contiguous(), shift.contiguous()


def tail_reference(skip, coarse, idx, out_rows_per_batch, src_rows_per_batch, ws, scale, shift, classes):
    """float64: x0 = [skip | coarse[row]] where row = idx (global) or idx + (n / out_rows_per_batch) * src_rows_per_batch
    (batch-relative); x0's coarse half is zero when idx < 0, idx >= src_rows_per_batch (batch-relative) or the row is
    not below coarse_rows.  Then three SharedMLPs (scale, shift, LeakyReLU) and the classifier (scale, shift)."""
    s = skip.double().cpu()
    c = coarse.double().cpu()
    n = s.shape[0]
    r = idx.cpu().long().clone()
    valid = r >= 0
    if out_rows_per_batch > 0:
        valid &= r < src_rows_per_batch
        r = r + torch.arange(n) // out_rows_per_batch * src_rows_per_batch
    valid &= r < c.shape[0]
    x = torch.cat([s, torch.where(valid.unsqueeze(1), c[r.clamp(0, c.shape[0] - 1)], torch.zeros(n, 32,
                                                                                                   dtype=torch.float64))], 1)
    lrelu = torch.nn.functional.leaky_relu
    for li, w in enumerate(ws):
        k, m = w.shape
        x = x @ w.double() * scale[li, :m].double() + shift[li, :m].double()
        if li < 3:
            x = lrelu(x, SLOPE)
    return x


def run_tail(skip, coarse, idx, orpb, srpb, rows, img, scale, shift, classes, pad=PAD):
    """One launch into a NaN-filled [rows + pad, classes] output."""
    out = torch.full(((rows + pad) * classes,), NAN).cuda()
    L.check(L.lib().o3dml_randla_tail(L.ptr(skip), skip.stride(0), L.ptr(coarse), coarse.stride(0), coarse.shape[0],
                                      L.ptr(idx), 1 if idx.dtype == torch.int64 else 0, orpb, srpb, rows, L.ptr(img),
                                      scale.data_ptr(), shift.data_ptr(), SLOPE, classes, L.ptr(out), L.stream()))
    torch.cuda.synchronize()
    return out


def assert_bounds(out, n):
    assert bool(torch.isfinite(out[:n]).all()), "unwritten or non-finite logits"
    assert bool((bits(out[n:]) == bits(torch.tensor(NAN)).item()).all()), "a sentinel was written"


def bits(t):
    """Bitwise view for torch.equal: the NaN sentinels compare equal to themselves."""
    return t.view(torch.int32)


def columns(rows, ch, ld, seed, mag=1.0):
    """[rows, ch] column view of a wider [rows, ld] buffer (row stride ld)."""
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(rows, ld, generator=g) * mag).cuda()[:, :ch]


def interp_index(rows, orpb, srpb, coarse_rows, dtype, seed):
    """Valid rows, with about 3 % each of -1, src_rows_per_batch (batch-relative) / coarse_rows (global) and
    coarse_rows + 5: every one of these selects no coarse row."""
    g = torch.Generator().manual_seed(seed)
    hi = srpb if orpb > 0 else coarse_rows
    idx = torch.randint(0, hi, (rows,), generator=g)
    u = torch.rand(rows, generator=g)
    idx[u < 0.03] = -1
    idx[(u >= 0.03) & (u < 0.06)] = hi
    idx[(u >= 0.06) & (u < 0.09)] = coarse_rows + 5
    return idx.to(dtype).cuda()


def case(rows, classes, dtype, batch_rel, ld, seed, mag=1.0, bn=True):
    """Inputs of one tail call: batch-relative indices use out_rows_per_batch = 300 (the last batch item may be
    partial) and src_rows_per_batch = 77."""
    orpb, srpb = (300, 77) if batch_rel else (0, 0)
    coarse_rows = ((rows + 299) // 300) * 77 if batch_rel else max(rows // 4, 1)
    skip = columns(rows, 32, ld, seed, mag)
    coarse = columns(coarse_rows, 32, ld, seed + 1, mag)
    idx = interp_index(rows, orpb, srpb, coarse_rows, dtype, seed + 2)
    ws, scale, shift = make_weights(classes, seed + 3, bn)
    img = L.pack_tail_image(ws, [32, 64, 32, 32]).cuda()
    return skip, coarse, idx, orpb, srpb, ws, scale, shift, img


# Largest float64 errors measured on an H100 80GB HBM3 over the cases of test_tail_vs_float64: rel_err 6.0e-6,
# elem_err 2.6e-4; of test_tail_is_magnitude_independent: rel_err 1.9e-6.  The bounds are about 5x those.
TOL_REL, TOL_ELEM = 3e-5, 1.3e-3


def rows_list():
    return [1, 127, 128, 129, 2 * sms() * 128 + 77]


@pytest.mark.parametrize("classes", [1, 8, 13, 19, 32])
@pytest.mark.parametrize("ri", range(5), ids=["r1", "r127", "r128", "r129", "r2S128+77"])
@pytest.mark.parametrize("dtype,batch_rel,ld", [(torch.int64, True, 32), (torch.int32, False, 36),
                                                (torch.int64, False, 48), (torch.int32, True, 48)],
                         ids=["i64-rel-ld32", "i32-glob-ld36", "i64-glob-ld48", "i32-rel-ld48"])
def test_tail_vs_float64(classes, ri, dtype, batch_rel, ld):
    rows = rows_list()[ri]
    skip, coarse, idx, orpb, srpb, ws, scale, shift, img = case(rows, classes, dtype, batch_rel, ld,
                                                                 classes * 1000 + ri * 10 + ld)
    want = tail_reference(skip, coarse, idx, orpb, srpb, ws, scale, shift, classes)
    out = run_tail(skip, coarse, idx, orpb, srpb, rows, img, scale, shift, classes)
    assert_bounds(out, rows * classes)
    got = out[:rows * classes].view(rows, classes)
    re, ee = rel_err(got, want), elem_err(got, want)
    assert re < TOL_REL and ee < TOL_ELEM, (re, ee)


def test_tail_invalid_indices_zero_the_coarse_half():
    """-1, src_rows_per_batch and coarse_rows give the same logits as an all-zero coarse row."""
    rows, classes = 512, 13
    skip, coarse, idx, orpb, srpb, ws, scale, shift, img = case(rows, classes, torch.int64, True, 32, 11)
    zero = torch.zeros(1, 32).cuda()
    zi = torch.zeros(rows, dtype=torch.int64).cuda()
    b = run_tail(skip, zero, zi, 0, 0, rows, img, scale, shift, classes)
    assert_bounds(b, rows * classes)
    for o, s, bad in ((orpb, srpb, -1), (orpb, srpb, srpb), (orpb, srpb, 1 << 40),
                      (0, 0, -1), (0, 0, coarse.shape[0]), (0, 0, 1 << 40)):
        bi = torch.full((rows,), bad, dtype=torch.int64).cuda()
        a = run_tail(skip, coarse, bi, o, s, rows, img, scale, shift, classes)
        assert torch.equal(bits(a), bits(b)), (o, bad)


@pytest.mark.parametrize("mag", [1e-20, 1e-6, 1e-3, 1.0, 3e4, 1e20])
def test_tail_is_magnitude_independent(mag):
    """3xTF32 keeps fp32's exponent: with zero shifts the four layers are positively homogeneous, and the relative
    error must not depend on the scale of the inputs."""
    rows, classes = 1000, 19
    skip, coarse, idx, orpb, srpb, ws, scale, shift, img = case(rows, classes, torch.int64, True, 32, 21, mag, bn=False)
    want = tail_reference(skip, coarse, idx, orpb, srpb, ws, scale, shift, classes)
    got = run_tail(skip, coarse, idx, orpb, srpb, rows, img, scale, shift, classes)[:rows * classes].view(rows, classes)
    re = rel_err(got, want)
    assert re < TOL_REL, re


def test_tail_output_is_schedule_invariant():
    """A row's logits depend on its own inputs and the weights only: bitwise the same alone, behind P prefix rows
    (P / 128 in 1, 2, 3, S - 1, S, S + 1, 2S + 3), with int32 instead of int64 indices, and launched twice."""
    S = sms()
    nb, classes = 3 * 128 + 77, 19
    skip, coarse, idx, _, _, ws, scale, shift, img = case(nb, classes, torch.int64, False, 32, 31)
    alone = run_tail(skip, coarse, idx, 0, 0, nb, img, scale, shift, classes)
    n = nb * classes
    assert_bounds(alone, n)
    assert torch.equal(bits(run_tail(skip, coarse, idx, 0, 0, nb, img, scale, shift, classes)), bits(alone))
    assert torch.equal(bits(run_tail(skip, coarse, idx.to(torch.int32), 0, 0, nb, img, scale, shift, classes)),
                       bits(alone))
    for pt in (1, 2, 3, S - 1, S, S + 1, 2 * S + 3):
        P = pt * 128
        g = torch.Generator().manual_seed(pt)
        ps = torch.cat([torch.randn(P, 32, generator=g).cuda(), skip])
        pi = torch.cat([torch.randint(0, coarse.shape[0], (P,), generator=g).cuda(), idx])
        out = run_tail(ps, coarse, pi, 0, 0, P + nb, img, scale, shift, classes)
        assert_bounds(out, (P + nb) * classes)
        assert torch.equal(out[P * classes:(P + nb) * classes], alone[:n]), pt


def tail_call(classes=13, skip_ld=48, coarse_ld=48, img=True, rows=256):
    skip, coarse, idx, orpb, srpb, ws, scale, shift, im = case(max(rows, 1), 13, torch.int64, True, 48, 41)
    out = torch.full(((rows + PAD) * 33,), NAN).cuda()
    rc = L.lib().o3dml_randla_tail(L.ptr(skip), skip_ld, L.ptr(coarse), coarse_ld, coarse.shape[0], L.ptr(idx), 1,
                                   orpb, srpb, rows, L.ptr(im) if img else None, scale.data_ptr(), shift.data_ptr(),
                                   SLOPE, classes, L.ptr(out), L.stream())
    torch.cuda.synchronize()
    return rc, out


@pytest.mark.parametrize("kw", [dict(classes=0), dict(classes=33), dict(skip_ld=50), dict(coarse_ld=46),
                                dict(img=False)], ids=["classes0", "classes33", "skip_ld50", "coarse_ld46", "no_image"])
def test_tail_rejects_bad_arguments(kw):
    n0 = L.lib().o3dml_launch_count()
    rc, out = tail_call(**kw)
    assert rc != 0
    with pytest.raises(RuntimeError):
        L.check(rc)
    assert L.lib().o3dml_launch_count() == n0
    assert bool(out.isnan().all())


def test_tail_zero_rows_launches_nothing():
    n0 = L.lib().o3dml_launch_count()
    rc, out = tail_call(rows=0)
    assert rc == 0 and L.lib().o3dml_launch_count() == n0
    assert bool(out.isnan().all())
