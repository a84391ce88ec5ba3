"""KPConv's neighbour gather + kernel-point correlation (pool.cu o3dml_kpconv_gather) against the torch port's gather
(oracle/models_torch.kp_gather) in float64, and the index max pool (o3dml_gather_max) against a restatement, at every
kernel instantiation the entry dispatches to and at the index, shape and scheduling edges where such kernels go
wrong."""
import pytest
import torch

from open3d_ml_b200 import _lib as L
from oracle import models_torch as MT

from conftest import rel_err

EXTENT = 0.125
# Against float64 on an H100 80GB HBM3 (400 W power limit), the largest rel_err of the gathered tensor over all cases
# below was 2.25e-7; the bound keeps about 5x of margin.
KPG_TOL = 1.2e-6


# in_channels, byte offset of the feature rows -> the lanes that share one query in the kernel the entry runs: the
# grouped kernels <LPQ, NE> <8,1>, <8,4>, <16,4>, <32,4>, then the shuffle kernel (a whole warp) with NE = 1, 2, 4 and,
# for rows that are not 16-byte aligned, 2.  test_gpu_launch_count.py checks these choices in a profiler trace.
DISPATCH = {(5, 0): 8, (32, 0): 8, (64, 0): 16, (256, 0): 32, (10, 0): 32, (50, 0): 32, (130, 0): 32, (64, 4): 32}


def _case(cin, H, K, nq, ns=300, offset=0, int32=False, seed=0):
    """Inputs with every id form: ids -1 and ns, query 1 all shadow (when nq > 1), per-query valid prefixes of different
    lengths followed by shadow tails, a neighbour exactly on kernel point 0 of query 0 and one exactly `extent` away
    from it."""
    g = torch.Generator().manual_seed(seed)
    s = (torch.rand(ns, 3, generator=g) - 0.5) * 0.3
    q = (torch.rand(nq, 3, generator=g) - 0.5) * 0.3
    kp = (torch.rand(K, 3, generator=g) - 0.5) * 0.3
    q[0] = 0.0
    kp[0] = torch.tensor([0.0625, -0.03125, 0.015625])
    s[0] = kp[0]                                                     # influence 1 on kernel point 0
    s[1] = kp[0] + torch.tensor([EXTENT, 0.0, 0.0])                  # influence 0 on kernel point 0
    nb = torch.randint(0, ns, (nq, H), generator=g)
    if H:
        shadow = torch.rand(nq, H, generator=g) < 0.1
        nb[shadow] = torch.where(torch.rand(nq, H, generator=g) < 0.5, -1, ns)[shadow]
        tail = torch.randint(0, H + 1, (nq,), generator=g)              # valid prefix length per query
        pos = torch.arange(H).view(1, -1)
        nb = torch.where(pos >= tail.view(-1, 1), torch.where(pos % 2 == 0, ns, -1), nb)
        nb[0, 0] = 0
        if H > 1:
            nb[0, 1] = 1
        if nq > 1:
            nb[1] = torch.where(pos[0] % 3 == 0, -1, ns)
    nb = nb.to(torch.int32 if int32 else torch.int64)
    store = torch.randn(ns * cin + 4, generator=g).cuda()
    x = store[offset // 4:offset // 4 + ns * cin].view(ns, cin)
    return q.cuda(), s.cuda(), nb.cuda(), x, kp.cuda()


def _run(q, s, nb, x, kp, extent, out):
    return L.lib().o3dml_kpconv_gather(L.ptr(q), q.shape[0], L.ptr(s), s.shape[0], L.ptr(nb), L.is64(nb), nb.shape[1],
                                       L.ptr(x), x.shape[1], L.ptr(kp), kp.shape[0], extent, L.ptr(out), L.stream())


def kpconv_gather_errors(cin, offset, int32):
    """rel_err of every (K, H, nq) case of one dispatch; the output rows past nq start as NaN and must keep it."""
    lpq = DISPATCH[(cin, offset)]
    errs = {}
    for K in (1, 15, 16):
        for H in sorted({0, 1, lpq - 1, lpq + 1, 32, 33, 65}):
            for nq in (1, 77):
                q, s, nb, x, kp = _case(cin, H, K, nq, offset=offset, int32=int32, seed=K * 1000 + H * 10 + nq)
                out = torch.full((nq + 5, K * cin), float("nan")).cuda()
                L.check(_run(q, s, nb, x, kp, EXTENT, out))
                ref = MT.kp_gather(q.double(), s.double(), nb, x.double(), kp.double(), EXTENT).flatten(1)
                assert bool(out[nq:].isnan().all()), (K, H, nq)
                errs[(K, H, nq)] = rel_err(out[:nq], ref)
    return errs


@pytest.mark.gpu
@pytest.mark.parametrize("int32", [False, True])
@pytest.mark.parametrize("cin,offset", list(DISPATCH))
def test_kpconv_gather_vs_float64(cin, offset, int32):
    errs = kpconv_gather_errors(cin, offset, int32)
    worst = max(errs, key=errs.get)
    assert errs[worst] < KPG_TOL, (worst, errs[worst])


@pytest.mark.gpu
@pytest.mark.parametrize("K,H,extent", [(0, 8, EXTENT), (17, 8, EXTENT), (15, 8, 0.0), (15, 8, -1.0), (15, -1, EXTENT)])
def test_kpconv_gather_rejects_without_launch(K, H, extent):
    q, s, nb, x, kp = _case(32, 8, 16, 10)
    kp = torch.zeros(max(K, 1), 3).cuda()[:K]
    out = torch.full((10, 16 * 32), float("nan")).cuda()
    n0 = L.lib().o3dml_launch_count()
    rc = L.lib().o3dml_kpconv_gather(L.ptr(q), 10, L.ptr(s), s.shape[0], L.ptr(nb), 1, H, L.ptr(x), 32, L.ptr(kp), K,
                                     extent, L.ptr(out), L.stream())
    assert rc != 0 and L.lib().o3dml_launch_count() == n0
    with pytest.raises(RuntimeError):
        L.check(rc)
    assert bool(out.isnan().all())


# ------------------------------------------------------------------------------------------------------ gather_max
def gather_max_reference(x, idx, shadow_zero, out_rows_per_batch=0, src_rows_per_batch=0):
    """out[n] = max over the valid ids of row n (ids in [0, rows), batch-relative when out_rows_per_batch > 0); invalid
    ids take part as a zero row when shadow_zero, else they are skipped; a row with nothing to take is zero."""
    n, k = idx.shape
    r = idx.long()
    if out_rows_per_batch > 0:
        ok = (r >= 0) & (r < src_rows_per_batch)
        r = r + (torch.arange(n, device=r.device) // out_rows_per_batch).view(-1, 1) * src_rows_per_batch
    else:
        ok = (r >= 0) & (r < x.shape[0])
    pad = torch.zeros(1, x.shape[1], device=x.device) if shadow_zero else torch.full((1, x.shape[1]), -float("inf"),
                                                                                      device=x.device)
    xp = torch.cat([x, pad])
    v = xp[torch.where(ok, r, x.shape[0])].amax(1)
    if not shadow_zero:
        v[~ok.any(1)] = 0.0
    return v


GMAX_CASES = ["batched", "global_shadow_zero", "global_skip", "k1_closest", "neg_inf", "very_negative"]


@pytest.mark.gpu
@pytest.mark.parametrize("int32", [False, True])
@pytest.mark.parametrize("case", GMAX_CASES)
def test_gather_max_bit_exact(case, int32):
    g = torch.Generator().manual_seed(GMAX_CASES.index(case))
    C, ld, rows = 24, 28, 500
    wide = torch.randn(rows, ld, generator=g)
    if case == "neg_inf":                   # rows of -inf, and -inf mixed into others
        wide[:50] = -float("inf")
        wide[50:100, ::3] = -float("inf")
    if case == "very_negative":
        wide = -wide.abs() * 3e38
    x = wide.cuda()[:, 4:4 + C]                                          # a column slice: ld > channels, 16-byte aligned
    n, k, orpb, srpb, sz = 300, 7, 0, 0, 0
    if case == "k1_closest":
        k = 1
    idx = torch.randint(-1, rows + 1, (n, k), generator=g)
    if case == "batched":
        orpb, srpb = 150, 250
        idx = torch.randint(-1, srpb + 2, (n, k), generator=g)
    if case in ("global_shadow_zero", "very_negative", "neg_inf"):
        sz = 1
    idx[0] = -1                                                          # nothing valid
    idx[1] = rows if not orpb else srpb
    if case == "neg_inf":
        idx[2] = torch.arange(k) % 50                                    # only -inf rows
        sz = 0
    idx = idx.to(torch.int32 if int32 else torch.int64).cuda()
    out = torch.full((n, C + 8), float("nan")).cuda()
    dst = out[:, 4:4 + C]
    n0 = L.lib().o3dml_launch_count()
    L.check(L.lib().o3dml_gather_max(L.ptr(x), rows, C, ld, L.ptr(idx), L.is64(idx), n, k, orpb, srpb, sz, L.ptr(dst),
                                     C + 8, L.stream()))
    assert L.lib().o3dml_launch_count() == n0 + 1
    ref = gather_max_reference(x, idx, sz, orpb, srpb)
    assert torch.equal(dst, ref)
    assert bool(out[:, :4].isnan().all()) and bool(out[:, 4 + C:].isnan().all())
    if not sz:
        assert float(dst[0].abs().max()) == 0 and float(dst[1].abs().max()) == 0
    if case == "neg_inf":
        assert bool((dst[2] == -float("inf")).all())
