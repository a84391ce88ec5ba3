"""Float64 torch port of the reference SparseConvUnet forward (ml3d/torch/models/sparseconvnet.py:73-93, 286-657),
built from a state_dict, and the lattice rules of DESIGN.md section 2 ("SparseConvUnet") in numpy.

The port computes what the unmodified class computes, item by item, in float64:
  * InputLayer: one voxel per occupied unit cell k = floor(p); its feature is the mean of its points' features; a
    point's output row is its voxel's.
  * SubmanifoldSparseConv (3^3, offset 0): out[v] = sum over the 27 cells (x slowest, z fastest) of W_cell^T x[u],
    u the voxel at k_v + cell - 1; an empty cell adds nothing.
  * Convolution (2^3, offset -0.5) onto calculate_grid's coarse lattice: voxel v adds W_{k mod 2}^T x[v] to its
    parent floor(k / 2); DeConvolution: voxel v gets W_{k mod 2}^T x[parent(v)].
  * BatchNormBlock (eval, eps 1e-4), ReLU, NetworkInNetwork, ResidualBlock, JoinFeat, LinearBlock, OutputLayer.
Voxel order inside a level is lexicographic here; no output depends on it."""
import numpy as np
import torch

BN_EPS = 1e-4


def unit_cells(points):
    """int64 [N, 3] cells k = floor(p) of float points."""
    return np.floor(np.asarray(points, np.float64)).astype(np.int64)


def np_voxels(k):
    """Unique cells of k [N, 3] (lexicographic) and each row's voxel."""
    return np.unique(k, axis=0, return_inverse=True)


def np_parent_cell(k):
    """Per fine voxel at cells k [M, 3]: the coarse lattice (unique floor(k / 2)), the parent's row in it and the
    kernel cell ((kx mod 2) * 2 + ky mod 2) * 2 + kz mod 2 of the 2^3 convolutions."""
    coarse, parent = np.unique(k // 2, axis=0, return_inverse=True)
    c = k & 1
    return coarse, parent.reshape(-1), (c[:, 0] * 2 + c[:, 1]) * 2 + c[:, 2]


def np_calculate_grid_parent_cell(pos, offset=-0.5):
    """What the reference's own float positions give: calculate_grid (sparseconvnet.py:388-401) of pos and, per input,
    the coarse row and the 2^3 cell floor(in - out + offset + 1) of the strided convolution."""
    k = np.floor(pos).astype(np.int64)
    cand = (k[:, None, :] + np.array([[a, b, c] for a in (-1, 0) for b in (-1, 0) for c in (-1, 0)])[None]).reshape(-1, 3)
    cand = cand[(cand.min(1) >= 0) & ~(cand % 2).astype(bool).any(1)]
    out = np.unique(cand, axis=0) + 0.5
    cell = np.floor(pos[:, None, :] - out[None] + offset + 1.0)
    inside = ((cell >= 0) & (cell < 2)).all(2)
    row = inside.argmax(1)
    assert inside.sum(1).max() == 1 and inside.any(1).all()
    c = cell[np.arange(len(pos)), row].astype(np.int64)
    return out, row, (c[:, 0] * 2 + c[:, 1]) * 2 + c[:, 2]


def np_sub_table(k):
    """[M, 27] rows of the voxel at k + cell - 1 per 3^3 cell (x slowest), M for an empty cell."""
    m = len(k)
    base = k.min(0) - 1
    ext = k.max(0) - base + 2
    key = ((k[:, 0] - base[0]) * ext[1] + (k[:, 1] - base[1])) * ext[2] + (k[:, 2] - base[2])
    order = np.argsort(key)
    sk = key[order]
    out = np.full((m, 27), m, np.int64)
    c = 0
    for dx in (-1, 0, 1):
        for dy in (-1, 0, 1):
            for dz in (-1, 0, 1):
                q = key + (dx * ext[1] + dy) * ext[2] + dz
                j = np.clip(np.searchsorted(sk, q), 0, m - 1)
                hit = sk[j] == q
                out[hit, c] = order[j[hit]]
                c += 1
    return out


def _bn_relu(sd, prefix, x):
    s = sd[prefix + ".weight"].double() / torch.sqrt(sd[prefix + ".running_var"].double() + BN_EPS)
    return torch.relu((x - sd[prefix + ".running_mean"].double()) * s + sd[prefix + ".bias"].double())


def _sub(x, table, w):
    """3^3 submanifold convolution: w [3, 3, 3, Cin, Cout]."""
    w = w.double().reshape(27, w.shape[-2], w.shape[-1])
    xp = torch.cat([x, x.new_zeros(1, x.shape[1])])
    out = x.new_zeros(x.shape[0], w.shape[2])
    for c in range(27):
        out += xp[table[:, c]] @ w[c]
    return out


def _down(x, parent, cell, mc, w):
    w = w.double().reshape(8, w.shape[-2], w.shape[-1])
    out = x.new_zeros(mc, w.shape[2])
    for c in range(8):
        sel = cell == c
        out.index_add_(0, parent[sel], x[sel] @ w[c])
    return out


def _up(x, parent, cell, w):
    w = w.double().reshape(8, w.shape[-2], w.shape[-1])
    out = x.new_zeros(len(parent), w.shape[2])
    for c in range(8):
        sel = cell == c
        out[sel] = x[parent[sel]] @ w[c]
    return out


def sparseconvunet_item(sd, cfg, points, feat, device="cpu"):
    """Logits [N, classes] of one item (points [N, 3] inside [0, grid_size), feat [N, 3])."""
    dev = torch.device(device)
    m = int(cfg["multiplier"])
    reps, residual = int(cfg.get("conv_block_reps", 1)), bool(cfg.get("residual_blocks", False))
    planes = [m * (i + 1) for i in range(7)]
    sd = {k: v.to(dev) for k, v in sd.items()}
    k0 = unit_cells(points)
    vox, inv = np_voxels(k0)
    f = torch.as_tensor(np.asarray(feat, np.float64), device=dev)
    cnt = torch.zeros(len(vox), dtype=torch.float64, device=dev).index_add_(
        0, torch.as_tensor(inv.reshape(-1), device=dev), torch.ones(len(inv), dtype=torch.float64, device=dev))
    x = torch.zeros(len(vox), 3, dtype=torch.float64, device=dev).index_add_(
        0, torch.as_tensor(inv.reshape(-1), device=dev), f) / cnt[:, None]
    lattice = [vox]
    while len(lattice) < 7:
        lattice.append(np_parent_cell(lattice[-1])[0])
    sub = [torch.as_tensor(np_sub_table(k), device=dev) for k in lattice]
    links = [None] + [tuple(torch.as_tensor(a, device=dev) for a in np_parent_cell(lattice[l - 1])[1:])
                      for l in range(1, 7)]
    x = _sub(x, sub[0], sd["sub_sparse_conv.net.kernel"])
    idx = [0]

    def key(suffix):
        return "unet.net.%d.%s" % (idx[0], suffix)

    def block(x, l, a, b):
        if residual:
            h = _sub(_bn_relu(sd, key("batch_norm1.bn"), x), sub[l], sd[key("sub_sparse_conv1.net.kernel")])
            h = _sub(_bn_relu(sd, key("batch_norm2.bn"), h), sub[l], sd[key("sub_sparse_conv2.net.kernel")])
            lin = x if a == b else x @ sd[key("lin.linear.weight")].double().t()
            idx[0] += 1
            return lin + h
        h = _bn_relu(sd, key("bn"), x)
        idx[0] += 2
        h = _sub(h, sub[l], sd[key("net.kernel")])
        idx[0] += 1
        return h

    def unet(x, l):
        for _ in range(reps):
            x = block(x, l, planes[l], planes[l])
        if l + 1 < 7:
            skip = x
            idx[0] += 1                                  # ConcatFeat
            h = _bn_relu(sd, key("bn"), x)
            idx[0] += 2
            parent, cell = links[l + 1]
            h = _down(h, parent, cell, len(lattice[l + 1]), sd[key("net.kernel")])
            idx[0] += 1
            h = unet(h, l + 1)
            h = _bn_relu(sd, key("bn"), h)
            idx[0] += 2
            h = _up(h, parent, cell, sd[key("net.kernel")])
            idx[0] += 2                                  # DeConvolution, JoinFeat
            x = torch.cat([skip, h], 1)
            for i in range(reps):
                x = block(x, l, planes[l] * (2 if i == 0 else 1), planes[l])
        return x
    x = unet(x, 0)
    x = _bn_relu(sd, "batch_norm.bn", x)
    x = x @ sd["linear.linear.weight"].double().t() + sd["linear.linear.bias"].double()
    return x[torch.as_tensor(inv.reshape(-1), device=dev)]


def sparseconvunet_forward(sd, batch, cfg, device="cpu"):
    """SparseConvUnet.forward of a SparseConvUnetBatch-like object (point, feat lists): [sum N_i, classes]."""
    return torch.cat([sparseconvunet_item(sd, cfg, p.detach().cpu().numpy(), f.detach().cpu().numpy(), device)
                      for p, f in zip(batch.point, batch.feat)])


def seeded_state_dict(cfg, seed=0, shift_bias=0.0):
    """A SparseConvUnet state_dict (the reference's keys and shapes) with seeded weights and randomised BN statistics;
    shift_bias moves every BN bias up, so that relu(BN(0)) > 0 (what an empty cell must NOT contribute)."""
    g = torch.Generator().manual_seed(seed)
    m = int(cfg["multiplier"])
    reps, residual = int(cfg.get("conv_block_reps", 1)), bool(cfg.get("residual_blocks", False))
    planes = [m * (i + 1) for i in range(7)]
    sd = {}

    def conv(prefix, ks, a, b):
        sd[prefix + ".kernel"] = (torch.rand(ks, ks, ks, a, b, generator=g) * 2 - 1) * (3.0 / (ks ** 3 * a)) ** 0.5
        sd[prefix + ".offset"] = torch.full((3,), 0.0 if ks == 3 else -0.5)

    def bn(prefix, c):
        sd[prefix + ".weight"] = 0.5 + torch.rand(c, generator=g)
        sd[prefix + ".bias"] = torch.randn(c, generator=g) * 0.1 + shift_bias
        sd[prefix + ".running_mean"] = torch.randn(c, generator=g) * 0.1
        sd[prefix + ".running_var"] = 0.5 + torch.rand(c, generator=g)
        sd[prefix + ".num_batches_tracked"] = torch.tensor(0)

    conv("sub_sparse_conv.net", 3, 3, m)
    i = [0]

    def block(a, b):
        p = "unet.net.%d" % i[0]
        if residual:
            if a != b:
                sd[p + ".lin.linear.weight"] = torch.randn(b, a, generator=g) / a ** 0.5
            bn(p + ".batch_norm1.bn", a)
            conv(p + ".sub_sparse_conv1.net", 3, a, b)
            bn(p + ".batch_norm2.bn", b)
            conv(p + ".sub_sparse_conv2.net", 3, b, b)
            i[0] += 1
        else:
            bn(p + ".bn", a)
            conv("unet.net.%d.net" % (i[0] + 2), 3, a, b)
            i[0] += 3

    def unet(pl):
        for _ in range(reps):
            block(pl[0], pl[0])
        if len(pl) > 1:
            i[0] += 1
            bn("unet.net.%d.bn" % i[0], pl[0])
            conv("unet.net.%d.net" % (i[0] + 2), 2, pl[0], pl[1])
            i[0] += 3
            unet(pl[1:])
            bn("unet.net.%d.bn" % i[0], pl[1])
            conv("unet.net.%d.net" % (i[0] + 2), 2, pl[1], pl[0])
            i[0] += 4
            for r in range(reps):
                block(pl[0] * (2 if r == 0 else 1), pl[0])
    unet(planes)
    bn("batch_norm.bn", m)
    sd["linear.linear.weight"] = torch.randn(int(cfg.get("num_classes", 20)), m, generator=g) / m ** 0.5
    sd["linear.linear.bias"] = torch.randn(int(cfg.get("num_classes", 20)), generator=g) * 0.1
    return sd


class _OracleSparseConv(torch.nn.Module):
    """open3d.ml.torch.layers.SparseConv on the CPU oracle (oracle/ops.py c_sparse_conv, fp32): the constructor,
    `kernel` [kx, ky, kz, Cin, Cout] parameter, optional `bias` and `offset` buffer of the upstream layer."""
    TRANSPOSE = False

    def __init__(self, in_channels, filters, kernel_size, activation=None, use_bias=True, kernel_initializer=None,
                 bias_initializer=None, normalize=False, offset=None, **kwargs):
        super().__init__()
        ks = [int(k) for k in kernel_size]
        self.kernel = torch.nn.Parameter(torch.zeros(*ks, int(in_channels), int(filters)))
        self.bias = torch.nn.Parameter(torch.zeros(int(filters))) if use_bias else None
        if offset is None:
            offset = torch.zeros(3) if ks[0] % 2 else torch.full((3,), -0.5)
        self.register_buffer("offset", torch.as_tensor(offset, dtype=torch.float32).reshape(3).clone())
        self.normalize, self.activation = bool(normalize), activation

    def forward(self, inp_features, inp_positions, out_positions, voxel_size, **kwargs):
        from . import ops as O
        out = O.c_sparse_conv(inp_features.detach().numpy(), inp_positions.detach().numpy(),
                              out_positions.detach().numpy(), float(voxel_size), self.offset.numpy(),
                              self.kernel.detach().numpy(), None if self.bias is None else self.bias.detach().numpy(),
                              self.normalize, self.TRANSPOSE)
        out = torch.from_numpy(out)
        return self.activation(out) if self.activation is not None else out


class _OracleSparseConvTranspose(_OracleSparseConv):
    TRANSPOSE = True


def _oracle_reduce_subarrays_sum(values, row_splits):
    from . import ops as O
    return torch.from_numpy(O.c_reduce_subarrays_sum(values.detach().numpy(), row_splits.numpy()))


def bind_sparseconvunet():
    """For the golden recorder and the CPU tests: the unmodified reference module (sparseconvnet.py) with its
    SparseConv / SparseConvTranspose / reduce_subarrays_sum names bound to the CPU oracle in the imported module's
    globals (the shim's table leaves them unbound); its source stays as it is."""
    from . import refshim
    refshim.install()
    import ml3d.torch.models.sparseconvnet as ref
    ref.SparseConv, ref.SparseConvTranspose = _OracleSparseConv, _OracleSparseConvTranspose
    ref.reduce_subarrays_sum = _oracle_reduce_subarrays_sum
    return ref
