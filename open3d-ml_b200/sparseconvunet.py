"""SparseConvUnet forward on the sm_90a kernels: the fused replacement of ``SparseConvUnet.forward``
(ml3d/torch/models/sparseconvnet.py:73-93) and of the layers it calls (InputLayer :286-329, SubmanifoldSparseConv,
Convolution, DeConvolution :344-485, the UNet :567-657, BatchNormBlock / ReLUBlock / LinearBlock / OutputLayer).

The whole batch is one lattice: voxelize's batch row splits keep the items apart, and every convolution is ONE
table-mode tensor-core launch for all items (o3dml_sparse_conv_tc):

    level 0     voxelize(points, voxel 1, range [0, grid_size)) + the per-voxel mean of the features
    level l+1   voxelize(level-l cells, voxel 2): parent floor(k / 2) per axis, kernel cell k mod 2 of the 2^3
                convolutions; the down table [M_l+1, 8] and the up rows come from this grouping
    3^3 tables  one o3dml_sparse_conv_neighbors per level (offset 0, voxel 1), shared by every submanifold convolution
                of the level; items are spaced ITEM_SPACING cells apart along x so that they never meet
    BN -> ReLU -> conv   the folded BN and the ReLU are the contraction's prologue, which keeps empty cells at zero
    transposed 2^3       one launch on the coarse level into [M_coarse, 8 Cout]; fine voxel i reads row
                         parent(i) * 8 + cell(i) (a gather into its column slice of the join buffer)
    head        BN -> ReLU -> Linear as a one-cell contraction whose table is each point's voxel

One device-to-host read per forward: the level sizes and the count of points outside the grid, read after the pyramid.
Inference only.
"""
import itertools

import torch

from . import _lib as L
from . import layers as LY
from . import ops
from .pipeline import BufferCache

BN_EPS = 1e-4            # BatchNormBlock (sparseconvnet.py:229)
LEVELS = 7               # UNet planes m, 2m, ..., 7m (sparseconvnet.py:64-67)
ITEM_SPACING = 4100      # cells between batch items along x in the 3^3 searches: > grid_size + 1
MAX_KEY = 1 << 20        # the neighbour search keys hold |x| < 2^20 cells


def cfg_from_reference(cfg):
    """The reference's model section (sparseconvunet_scannet.yml) -> the keys SparseConvUnetB200 reads."""
    return dict(multiplier=int(cfg.get("multiplier", 16)), conv_block_reps=int(cfg.get("conv_block_reps", 1)),
                residual_blocks=bool(cfg.get("residual_blocks", False)), in_channels=int(cfg.get("in_channels", 3)),
                num_classes=int(cfg.get("num_classes", 20)), grid_size=int(cfg.get("grid_size", 4096)))


def unet_layout(planes, residual, reps):
    """UNet.get_UNet's module list (sparseconvnet.py:580-622) as tuples, in state_dict index order:
    ("res", a, b) | ("bn", c) | ("relu",) | ("sub", a, b) | ("concat",) | ("down", a, b) | ("up", a, b) | ("join",)."""
    out = []

    def block(a, b):
        out.extend([("res", a, b)] if residual else [("bn", a), ("relu",), ("sub", a, b)])
    for _ in range(reps):
        block(planes[0], planes[0])
    if len(planes) > 1:
        out.extend([("concat",), ("bn", planes[0]), ("relu",), ("down", planes[0], planes[1])])
        out.extend(unet_layout(planes[1:], residual, reps))
        out.extend([("bn", planes[1]), ("relu",), ("up", planes[1], planes[0]), ("join",)])
        for i in range(reps):
            block(planes[0] * (2 if i == 0 else 1), planes[0])
    return out


class SparseConvUnetB200:
    def __init__(self, state_dict, cfg, device=None):
        L.require_cuda()
        self.device = torch.device(device or "cuda")
        self.buf = BufferCache(self.device)
        self.cfg = cfg = dict(cfg)
        if int(cfg.get("in_channels", 3)) != 3:
            raise RuntimeError("SparseConvUnetB200: in_channels must be 3 (InputLayer writes three feature columns)")
        m = int(cfg["multiplier"])
        if m < 4 or m % 4:
            raise RuntimeError("SparseConvUnetB200: multiplier %d; the contraction reads feature rows whose width is a "
                               "multiple of 4 channels, so the multiplier must be one" % m)
        self.grid_size = int(cfg.get("grid_size", 4096))
        self.planes = [m * (i + 1) for i in range(LEVELS)]
        self.layout = unet_layout(self.planes, bool(cfg.get("residual_blocks", False)), int(cfg.get("conv_block_reps", 1)))
        sd = L.host_state_dict(state_dict)
        for k, v in sd.items():
            if k.endswith(".offset"):
                ks = sd[k[:-len("offset")] + "kernel"].shape[0]
                want = 0.0 if ks == 3 else -0.5
                if not bool((v == want).all()):
                    raise RuntimeError("SparseConvUnetB200: %s is %s; the %d^3 convolutions take offset %g"
                                       % (k, v.tolist(), ks, want))
        dev = self.device
        self.w = {}

        def put(name, t):
            self.w[name] = t.to(dev, torch.float32).contiguous()

        def bn(name, prefix):
            s, t = L.fold_bn(sd, prefix, BN_EPS)
            put(name + ".s", s), put(name + ".t", t)

        def conv(name, key):
            k = sd[key]
            self.w[name] = LY.pack_cells(k.reshape(-1, k.shape[-2], k.shape[-1]))

        w0 = sd["sub_sparse_conv.net.kernel"]
        if w0.shape[-2] != 3:
            raise RuntimeError("SparseConvUnetB200: the state_dict takes %d input channels, not 3" % w0.shape[-2])
        conv("in", "sub_sparse_conv.net.kernel")
        for i, spec in enumerate(self.layout):
            p = "unet.net.%d" % i
            if spec[0] == "bn":
                bn(p, p + ".bn")
            elif spec[0] == "sub":
                conv(p, p + ".net.kernel")
            elif spec[0] == "down":
                conv(p, p + ".net.kernel")
            elif spec[0] == "up":
                k = sd[p + ".net.kernel"].reshape(8, spec[1], spec[2])        # [cell, Cin, Cout]
                self.w[p] = LY.pack_cells(k.permute(1, 0, 2).reshape(1, spec[1], 8 * spec[2]))
            elif spec[0] == "res":
                bn(p + ".bn1", p + ".batch_norm1.bn")
                bn(p + ".bn2", p + ".batch_norm2.bn")
                conv(p + ".conv1", p + ".sub_sparse_conv1.net.kernel")
                conv(p + ".conv2", p + ".sub_sparse_conv2.net.kernel")
                if spec[1] != spec[2]:
                    self.w[p + ".lin"] = L.pack_linear(sd[p + ".lin.linear.weight"].t())
        bn("head", "batch_norm.bn")
        lw = sd["linear.linear.weight"]
        self.num_classes = lw.shape[0]
        self.w["head"] = LY.pack_cells(lw.t()[None])
        put("head.bias", sd["linear.linear.bias"])

    def rows(self, name, m, c, dtype=torch.float32):
        """A [m, c] buffer: the first m rows of a cached one whose row count is m rounded up to a power of two, so that
        scenes of varying size reuse a bounded set of buffers."""
        cap = 1 << max(10, (max(m, 1) - 1).bit_length())
        return self.buf.get(name, (cap, c), dtype)[:m]

    # ------------------------------------------------------------------ lattice
    def pyramid(self, points, splits):
        """Chained voxelize_raw over LEVELS levels, sizes still on the device.  Returns the per-level raw results and
        the one host read: [M_0 .. M_6, points outside the grid]."""
        n = points.shape[0]
        hi = torch.nextafter(torch.tensor(float(self.grid_size)), torch.tensor(0.0)).item()
        lv = [ops.voxelize_raw(points, splits, [1.0] * 3, [0.0] * 3, [hi] * 3, n, n, want_batch_id=True)]
        g = self.grid_size
        for _ in range(1, LEVELS):
            coords, _, _, bsp = lv[-1][:4]
            lv.append(ops.voxelize_raw(coords.float(), bsp, [2.0] * 3, [0.0] * 3, [float(g)] * 3, n, n,
                                       want_batch_id=True))
            g = (g + 1) // 2
        counts = torch.stack([r[5][0] for r in lv] + [n - lv[0][5][1]]).cpu().tolist()      # the one host read
        return lv, counts[:LEVELS], counts[LEVELS]

    def tables(self, lv, sizes):
        """Per level: the 3^3 table [M, 27]; per level l > 0: the down table [M_l, 8] and the up rows of level l - 1."""
        dev = self.device
        sub, down, up = [], [None], [None]
        for l, M in enumerate(sizes):
            coords, _, _, _, bid, _ = lv[l]
            pos = coords[:M].float() + 0.5
            pos[:, 0] += bid[:M].float() * ITEM_SPACING
            nbr, _ = LY.sparse_conv_neighbors(pos, pos, 1.0, [0.0, 0.0, 0.0], [3, 3, 3])
            sub.append(nbr)
            if l == 0:
                continue
            mf = sizes[l - 1]
            _, pidx, vrs = lv[l][:3]
            fine = torch.arange(mf, device=dev)
            parent = torch.empty(mf, dtype=torch.int64, device=dev)
            parent[pidx[:mf]] = torch.searchsorted(vrs[:M + 1], fine, right=True) - 1
            c = lv[l - 1][0][:mf].long() & 1
            cell = (c[:, 0] * 2 + c[:, 1]) * 2 + c[:, 2]
            d = torch.full((M, 8), mf, dtype=torch.int32, device=dev)
            d[parent, cell] = fine.to(torch.int32)
            down.append(d)
            up.append((parent * 8 + cell).to(torch.int32))
        return sub, down, up

    # ------------------------------------------------------------------ forward
    def forward(self, batch):
        dev = self.device
        if torch.is_grad_enabled() and any(t.requires_grad for t in list(batch.point) + list(batch.feat)):
            raise RuntimeError("open3d_ml_b200: the fused SparseConvUnet path is inference-only "
                               "(call under torch.no_grad())")
        pts = torch.cat([p.to(dev, torch.float32) for p in batch.point])
        feat = torch.cat([f.to(dev, torch.float32) for f in batch.feat])
        if feat.dim() != 2 or feat.shape[1] != 3:
            raise RuntimeError("SparseConvUnetB200: feat must be [N, 3]")
        lengths = [int(x) for x in batch.batch_lengths]
        n, B = pts.shape[0], len(lengths)
        if B < 1 or (B - 1) * ITEM_SPACING + self.grid_size >= MAX_KEY:
            raise RuntimeError("SparseConvUnetB200: 1..%d items per batch" % ((MAX_KEY - self.grid_size) // ITEM_SPACING))
        splits = torch.tensor(list(itertools.accumulate(lengths, initial=0)), dtype=torch.int64).pin_memory().to(
            dev, non_blocking=True)           # from pinned memory: no synchronising copy
        lv, sizes, outside = self.pyramid(pts, splits)
        if outside:
            raise RuntimeError("SparseConvUnetB200: %d points lie outside [0, %d)^3 (preprocess keeps them inside)"
                               % (outside, self.grid_size))
        if n == 0:
            return torch.empty((0, self.num_classes), dtype=torch.float32, device=dev)
        sub, down, up = self.tables(lv, sizes)
        # level 0: voxel position = its lowest-id point, feature = the fp32 mean of its points in ascending id
        _, pidx, vrs = lv[0][:3]
        f4 = self.rows("feat4", n, 4)
        f4[:, 3] = 0
        f4[:, :3] = feat
        x = self.rows("x0", sizes[0], 4)
        L.check(L.lib().o3dml_voxel_reduce(L.ptr(pts), 3, L.ptr(f4), 4, 4, None, L.ptr(vrs), L.ptr(pidx), None,
                                           sizes[0], 2, 0, None, L.ptr(x), None, L.stream()))
        voxel_of_point = torch.empty(n, dtype=torch.int32, device=dev)
        voxel_of_point[pidx[:n]] = (torch.searchsorted(vrs[:sizes[0] + 1], torch.arange(n, device=dev), right=True)
                                    - 1).to(torch.int32)
        x = self.conv(x[:, :3], sub[0], "in", self.rows("in.0", sizes[0], self.planes[0]))
        x = self.unet(x, sizes, sub, down, up)
        logits = torch.empty((n, self.num_classes), dtype=torch.float32, device=dev)
        LY.contract_cells(x, voxel_of_point.view(n, 1), self.w["head"], logits, self.w["head.bias"],
                          pre=(self.w["head.s"], self.w["head.t"]))
        return logits

    __call__ = forward

    def conv(self, x, table, name, out, pre=None, residual=None):
        return LY.contract_cells(x, table, self.w[name], out, pre=pre, residual=residual)

    def unet(self, x, sizes, sub, down, up):
        level, pre, skips = 0, None, []

        def fresh(l, c, avoid):
            """A level-l [M, c] buffer whose storage differs from every tensor in `avoid`."""
            for k in "pqr":
                t = self.rows("u.%d.%s" % (l, k), sizes[l], c)
                if all(t.data_ptr() != a.data_ptr() for a in avoid):
                    return t
            raise AssertionError("no free buffer")
        for i, spec in enumerate(self.layout):
            p = "unet.net.%d" % i
            kind = spec[0]
            to_skip = i + 1 < len(self.layout) and self.layout[i + 1][0] == "concat"

            def target(c, avoid):
                if to_skip:     # the encoder output is the left column slice of the level's join buffer
                    return self.rows("join.%d" % level, sizes[level], 2 * c)[:, :c]
                return fresh(level, c, avoid)
            if kind == "bn":
                pre = (self.w[p + ".s"], self.w[p + ".t"])
            elif kind == "relu":
                pass
            elif kind == "sub":
                x = self.conv(x, sub[level], p, target(spec[2], [x]), pre=pre)
                pre = None
            elif kind == "res":
                a, b = spec[1], spec[2]
                h = self.rows("h.%d" % level, sizes[level], b)
                self.conv(x, sub[level], p + ".conv1", h, pre=(self.w[p + ".bn1.s"], self.w[p + ".bn1.t"]))
                if a != b:
                    res = self.rows("lin.%d" % level, sizes[level], b)
                    L.linear([L.make_src(x)], self.w[p + ".lin"], res)
                else:
                    res = x
                x = self.conv(h, sub[level], p + ".conv2", target(b, [x]),
                              pre=(self.w[p + ".bn2.s"], self.w[p + ".bn2.t"]), residual=res)
            elif kind == "concat":
                skips.append(x)
            elif kind == "down":
                level += 1
                x = self.conv(x, down[level], p, fresh(level, spec[2], []), pre=pre)
                pre = None
            elif kind == "up":
                a, b = spec[1], spec[2]
                mc = sizes[level]
                ident = self.rows("ident", mc, 1, torch.int32)
                torch.arange(mc, dtype=torch.int32, device=self.device, out=ident.view(-1))
                u = self.rows("up.%d" % level, mc, 8 * b)
                self.conv(x, ident, p, u, pre=pre)
                pre = None
                rows = up[level]
                level -= 1
                skip = skips.pop()
                join = self.rows("join.%d" % level, sizes[level], 2 * b)
                assert skip.data_ptr() == join.data_ptr()
                L.check(L.lib().o3dml_gather_max(L.ptr(u), mc * 8, b, b, L.ptr(rows), 0, sizes[level], 1, 0, 0, 0,
                                                 L.ptr(join[:, b:]), 2 * b, L.stream()))
                x = join
            elif kind == "join":
                pass
        return x


def patch_reference_model(model):
    """Drop-in: make an (unmodified) reference ``SparseConvUnet`` instance run its forward on the fused CUDA path
    (keeps preprocess / transform / losses).  BN must be in eval mode."""
    fused = SparseConvUnetB200(model.state_dict(), cfg_from_reference(model.cfg))

    def forward(inputs):
        if model.training:
            raise RuntimeError("open3d_ml_b200: the fused SparseConvUnet path is inference-only")
        return fused.forward(inputs)
    model.forward = forward
    return model
