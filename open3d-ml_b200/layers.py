"""``open3d.ml.torch.layers.SparseConv`` / ``SparseConvTranspose`` on the sm_90a kernels
(call sites: ml3d/torch/models/sparseconvnet.py:344-485 -- SubmanifoldSparseConv, Convolution, DeConvolution of
SparseConvUnet).  Same constructor arguments and parameter names (``kernel`` [kx, ky, kz, Cin, Cout], ``bias``) as
the upstream layers, so reference checkpoints load; inference only (no autograd through the CUDA path).

forward = one neighbour-table kernel (o3dml_sparse_conv_neighbors: radix sort of the input voxels + one binary
search per (output, kernel cell)) followed by the gathered tensor-core GEMM with up to three kernel cells per
launch as index operands -- the [M, 27 * Cin] im2col tensor never exists.
"""
import numpy as np
import torch

from . import _lib as L


def sparse_conv_neighbors(inp_positions, out_positions, voxel_size, offset, kernel_size, transpose=False,
                          want_count=False):
    """int32 [M, kx*ky*kz] table (shadow id = N) and, optionally, the per-output count of non-empty cells."""
    L.require_cuda()
    ip = inp_positions.to("cuda", torch.float32).contiguous()
    op = out_positions.to("cuda", torch.float32).contiguous()
    n, m = ip.shape[0], op.shape[0]
    ks = np.asarray(kernel_size, dtype=np.int32).reshape(3)
    off = np.ascontiguousarray(torch.as_tensor(offset).detach().cpu().numpy(), dtype=np.float32).reshape(3)
    kc = int(ks.prod())
    nbr = torch.empty((m, kc), dtype=torch.int32, device=ip.device)
    cnt = torch.empty((m,), dtype=torch.int32, device=ip.device) if want_count else None
    wsb = L.lib().o3dml_sparse_conv_workspace_bytes(n)
    ws = torch.empty((wsb,), dtype=torch.uint8, device=ip.device)
    L.check(L.lib().o3dml_sparse_conv_neighbors(L.ptr(ip), n, L.ptr(op), m, float(voxel_size), off.ctypes.data,
                                                ks.ctypes.data, 1 if transpose else 0, L.ptr(nbr), L.ptr(cnt),
                                                L.ptr(ws), wsb, L.stream()))
    return nbr, cnt


def pack_cell_groups(w):
    """Kernel weights [cells, Cin, Cout] -> [(first cell, end cell, PackedWeight [cells * Cin, Cout])]: the cells
    grouped three at a time, one gathered GEMM each."""
    kc, cout = w.shape[0], w.shape[2]
    return [(a, min(a + 3, kc),L.pack_linear(w[a:a + 3].reshape(-1, cout))) for a in range(0, kc, 3)]


def contract_cells(feat, table, groups, out, bias=None):
    """out [M, Cout] = sum over the cells c of feat[table[:, c]] @ W_c, + bias: one gathered GEMM per group of
    pack_cell_groups, the first writing out (with the bias), the others adding onto it through their residual.
    table int32 [M, cells]; an empty cell holds the shadow id feat.shape[0]."""
    kc = table.shape[1]
    for gi, (a, b, pw) in enumerate(groups):
        srcs = [L.make_src(feat, index=table[:, c:], index_ld=kc) for c in range(a, b)]
        L.linear(srcs, pw, out, None, None if gi else bias, residual=out if gi else None, act=None)


class _SparseConvBase(torch.nn.Module):
    TRANSPOSE = False

    def __init__(self, in_channels, filters, kernel_size, activation=None, use_bias=True,
                 kernel_initializer=None, bias_initializer=None, normalize=False, offset=None, **kwargs):
        super().__init__()
        ks = [int(k) for k in kernel_size]
        if len(ks) != 3:
            raise RuntimeError("SparseConv: kernel_size must have 3 entries")
        self.in_channels, self.filters, self.kernel_size = int(in_channels), int(filters), ks
        self.activation, self.use_bias, self.normalize = activation, bool(use_bias), bool(normalize)
        if offset is None:      # upstream default: centred for odd kernels, shifted by half a voxel for even ones
            offset = torch.zeros(3) if ks[0] % 2 else torch.full((3,), -0.5)
        self.register_buffer("offset", torch.as_tensor(offset, dtype=torch.float32).reshape(3).clone())
        kernel = torch.empty(*ks, self.in_channels, self.filters)
        (kernel_initializer or (lambda t: torch.nn.init.uniform_(t, -0.05, 0.05)))(kernel)
        self.kernel = torch.nn.Parameter(kernel)
        if self.use_bias:
            bias = torch.zeros(self.filters)
            if bias_initializer is not None:
                bias_initializer(bias)
            self.bias = torch.nn.Parameter(bias)
        self._packed = None

    def _weights(self, dev):
        """pack_cell_groups of the kernel, cached per version."""
        key = (self.kernel._version, self.kernel.data_ptr(), str(dev))
        if self._packed is None or self._packed[0] != key:
            w = self.kernel.detach().reshape(-1, self.in_channels, self.filters).float().cpu()
            self._packed = (key, pack_cell_groups(w))
        return self._packed[1]

    def forward(self, inp_features, inp_positions, out_positions, voxel_size, inp_importance=None, **kwargs):
        if inp_importance is not None or kwargs.get("user_neighbors_index") is not None:
            raise RuntimeError("SparseConv: importance / user neighbours are not implemented")
        if torch.is_grad_enabled() and (inp_features.requires_grad or self.kernel.requires_grad and self.training):
            raise RuntimeError("open3d_ml_b200: SparseConv is inference-only (call under torch.no_grad() / eval())")
        L.require_cuda()
        ret_dev = inp_features.device
        feat = inp_features.detach().to("cuda", torch.float32).contiguous()
        n, m = feat.shape[0], out_positions.shape[0]
        vs = float(torch.as_tensor(voxel_size).reshape(-1)[0]) if not isinstance(voxel_size, (int, float)) else float(voxel_size)
        nbr, cnt = sparse_conv_neighbors(inp_positions, out_positions, vs, self.offset, self.kernel_size,
                                         self.TRANSPOSE, want_count=self.normalize)
        out = torch.zeros((m, self.filters), dtype=torch.float32, device=feat.device)
        if m and n:
            bias = self.bias.detach().to(feat.device, torch.float32) if self.use_bias and not self.normalize else None
            contract_cells(feat, nbr, self._weights(feat.device), out, bias)
        elif self.use_bias and not self.normalize:
            out += self.bias.detach().to(out.device)
        if self.normalize:
            out = out / cnt.clamp_min(1).to(torch.float32).unsqueeze(1)
            if self.use_bias:
                out = out + self.bias.detach().to(out.device)
        if self.activation is not None:
            out = self.activation(out)
        return out.to(ret_dev)


class SparseConv(_SparseConvBase):
    """open3d.ml.torch.layers.SparseConv: cell = floor((in - out) / voxel_size + offset + kernel_size / 2)."""
    TRANSPOSE = False


class SparseConvTranspose(_SparseConvBase):
    """open3d.ml.torch.layers.SparseConvTranspose: cell = floor((out - in) / voxel_size + offset + kernel_size / 2)."""
    TRANSPOSE = True


class ContinuousConv(torch.nn.Module):
    """open3d.ml.torch.layers.ContinuousConv: radius search (radius = extent / 2, in `radius_search_metric`, skipping
    points equal to the output point under `radius_search_ignore_query_points`) + ops.continuous_conv.  One extent:
    fixed_radius_search; one per output point: radius_search with those radii.  `window_function`, when given, maps
    the normalised distances (distance / (r * r) for L2, distance / r otherwise) to the neighbour importance.
    user_neighbors_index / _row_splits / _importance replace the search and the window.  kernel parameter
    [Sz, Sy, Sx, Cin, Cout] (`kernel`), optional `bias`; inference only."""

    def __init__(self, in_channels, filters, kernel_size, activation=None, use_bias=True, kernel_initializer=None,
                 bias_initializer=None, align_corners=True, coordinate_mapping="ball_to_cube_radial",
                 interpolation="linear", normalize=True, radius_search_ignore_query_points=False,
                 radius_search_metric="L2", offset=None, window_function=None, use_dense_layer_for_center=False,
                 **kwargs):
        super().__init__()
        if use_dense_layer_for_center:
            raise RuntimeError("ContinuousConv: use_dense_layer_for_center is not implemented")
        from . import ops
        ops._metric(radius_search_metric, "ContinuousConv")
        ks = [int(k) for k in kernel_size]
        self.in_channels, self.filters, self.kernel_size = int(in_channels), int(filters), ks
        self.activation, self.use_bias = activation, bool(use_bias)
        self.align_corners, self.coordinate_mapping = bool(align_corners), coordinate_mapping
        self.interpolation, self.normalize = interpolation, bool(normalize)
        self.radius_search_metric = radius_search_metric
        self.radius_search_ignore_query_points = bool(radius_search_ignore_query_points)
        self.window_function = window_function
        self.register_buffer("offset", torch.zeros(3) if offset is None else
                             torch.as_tensor(offset, dtype=torch.float32).reshape(3).clone())
        kernel = torch.empty(*ks, self.in_channels, self.filters)
        (kernel_initializer or (lambda t: torch.nn.init.uniform_(t, -0.05, 0.05)))(kernel)
        self.kernel = torch.nn.Parameter(kernel)
        if self.use_bias:
            bias = torch.zeros(self.filters)
            if bias_initializer is not None:
                bias_initializer(bias)
            self.bias = torch.nn.Parameter(bias)

    def _search(self):
        return dict(metric=self.radius_search_metric, ignore_query_point=self.radius_search_ignore_query_points)

    def forward(self, inp_features, inp_positions, out_positions, extents, inp_importance=None,
                user_neighbors_index=None, user_neighbors_row_splits=None, user_neighbors_importance=None, **kwargs):
        from . import ops
        ext = torch.as_tensor(extents, dtype=torch.float32).reshape(-1)
        window = self.window_function
        if user_neighbors_index is not None:
            if user_neighbors_row_splits is None:
                raise RuntimeError("ContinuousConv: user_neighbors_index needs user_neighbors_row_splits")
            idx, splits, importance = user_neighbors_index, user_neighbors_row_splits, user_neighbors_importance
        elif ext.numel() == 1:
            r = float(ext[0]) * 0.5
            res = ops.fixed_radius_search(inp_positions.float(), out_positions.float(), r,
                                          return_distances=window is not None, **self._search())
            idx, splits, importance = res.neighbors_index, res.neighbors_row_splits, None
            if window is not None:
                r32 = np.float32(r)
                scale = r32 * r32 if self.radius_search_metric == "L2" else r32
                importance = window(res.neighbors_distance / torch.tensor(scale, device=res.neighbors_distance.device))
        else:
            if ext.numel() != out_positions.shape[0]:
                raise RuntimeError("ContinuousConv: extents must have 1 or num_out elements")
            res = ops.radius_search(inp_positions.float(), out_positions.float(), ext * 0.5,
                                    return_distances=window is not None, normalize_distances=window is not None,
                                    **self._search())
            idx, splits, importance = res.neighbors_index, res.neighbors_row_splits, None
            if window is not None:
                importance = window(res.neighbors_distance)
        out = ops.continuous_conv(self.kernel.detach(), out_positions, ext, self.offset, inp_positions, inp_features,
                                  inp_importance, idx, importance, splits,
                                  self.align_corners, self.coordinate_mapping, self.normalize, self.interpolation)
        if self.use_bias:
            out = out + self.bias.detach().to(out.device)
        return self.activation(out) if self.activation is not None else out


class ContinuousConvTranspose(ContinuousConv):
    """open3d.ml.torch.layers.ContinuousConvTranspose: the constructor, parameters (`kernel` [Sz, Sy, Sx, Cin, Cout],
    `bias`) and `offset` buffer of ContinuousConv, so state_dicts load either way.  forward = one fixed-radius search
    of the outputs around each input (radius = extent / 2), ops.invert_neighbors_list of its lists and
    ops.continuous_conv_transpose; under `normalize` input i is scaled by 1 / its neighbour count.  One host read
    (the search's count); inference only."""

    def __init__(self, in_channels, filters, kernel_size, window_function=None, use_dense_layer_for_center=False,
                 **kwargs):
        if window_function is not None or use_dense_layer_for_center:
            raise RuntimeError("ContinuousConvTranspose: window_function and use_dense_layer_for_center are not "
                               "implemented")
        super().__init__(in_channels, filters, kernel_size, **kwargs)
        self._offset_host = None

    def _host_offset(self):
        """The `offset` buffer on the host, read once per version: the op takes it by value, and a module moved to
        the GPU would otherwise pay a device->host read per call."""
        key = (self.offset.data_ptr(), self.offset._version, str(self.offset.device))
        if self._offset_host is None or self._offset_host[0] != key:
            self._offset_host = (key, self.offset.detach().cpu())
        return self._offset_host[1]

    def forward(self, inp_features, inp_positions, out_positions, extents, out_importance=None, **kwargs):
        from . import ops
        for k in ("inp_neighbors_index", "inp_neighbors_importance_sum", "inp_neighbors_row_splits",
                  "user_neighbors_index", "user_neighbors_row_splits", "user_neighbors_importance"):
            if kwargs.get(k) is not None:
                raise RuntimeError("ContinuousConvTranspose: %s is not implemented (the layer runs its own search)" % k)
        ext = torch.as_tensor(extents, dtype=torch.float32).reshape(-1)
        if ext.numel() != 1:
            raise RuntimeError("ContinuousConvTranspose: one extent for all points (per-point extents: use "
                               "ops.continuous_conv_transpose)")
        ret_dev = inp_features.device
        op, ip = ops._dev(out_positions.float()), ops._dev(inp_positions.float())
        r = ops.fixed_radius_search(op, ip, float(ext[0]) * 0.5, return_distances=False, **self._search())
        inv = ops.invert_neighbors_list(op.shape[0], r.neighbors_index, r.neighbors_row_splits, torch.empty(0))
        out = ops.continuous_conv_transpose(self.kernel.detach(), op, out_importance, ext, self._host_offset(), ip,
                                            ops._dev(inp_features), r.neighbors_index, None, r.neighbors_row_splits,
                                            inv.neighbors_index, None, inv.neighbors_row_splits, self.align_corners,
                                            self.coordinate_mapping, self.normalize, self.interpolation)
        if self.use_bias:
            out = out + self.bias.detach().to(out.device)
        out = self.activation(out) if self.activation is not None else out
        return out.to(ret_dev)
