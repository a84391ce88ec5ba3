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
        """Kernel cells grouped three at a time into [3 * Cin, Cout] operands (PackedWeight), cached per version."""
        key = (self.kernel._version, self.kernel.data_ptr(), str(dev))
        if self._packed is None or self._packed[0] != key:
            kc = int(np.prod(self.kernel_size))
            w = self.kernel.detach().reshape(kc, self.in_channels, self.filters).float().cpu()
            groups = [(c0, min(c0 + 3, kc)) for c0 in range(0, kc, 3)]
            packs = [L.pack_linear(w[a:b].reshape((b - a) * self.in_channels, self.filters)) for a, b in groups]
            self._packed = (key, groups, packs)
        return self._packed[1], self._packed[2]

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
        kc = nbr.shape[1]
        out = torch.zeros((m, self.filters), dtype=torch.float32, device=feat.device)
        if m and n:
            groups, packs = self._weights(feat.device)
            bias = self.bias.detach().to(feat.device, torch.float32) if self.use_bias and not self.normalize else None
            for gi, ((a, b), pw) in enumerate(zip(groups, packs)):
                srcs = [L.make_src(feat, index=nbr[:, c:], index_ld=kc) for c in range(a, b)]
                L.linear(srcs, pw, out, None, bias if gi == 0 else None, residual=out if gi else None, act=None)
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
    """open3d.ml.torch.layers.ContinuousConv: fixed-radius search (radius = extent / 2) + ops.continuous_conv.
    kernel parameter [Sz, Sy, Sx, Cin, Cout] (`kernel`), optional `bias`; inference only."""

    def __init__(self, in_channels, filters, kernel_size, activation=None, use_bias=True, kernel_initializer=None,
                 bias_initializer=None, align_corners=True, coordinate_mapping="ball_to_cube_radial",
                 interpolation="linear", normalize=True, radius_search_ignore_query_points=False,
                 radius_search_metric="L2", offset=None, **kwargs):
        super().__init__()
        if radius_search_metric != "L2" or radius_search_ignore_query_points:
            raise RuntimeError("ContinuousConv: only the L2 radius search including the query point")
        ks = [int(k) for k in kernel_size]
        self.in_channels, self.filters, self.kernel_size = int(in_channels), int(filters), ks
        self.activation, self.use_bias = activation, bool(use_bias)
        self.align_corners, self.coordinate_mapping = bool(align_corners), coordinate_mapping
        self.interpolation, self.normalize = interpolation, bool(normalize)
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

    def forward(self, inp_features, inp_positions, out_positions, extents, inp_importance=None, **kwargs):
        from . import ops
        ext = torch.as_tensor(extents, dtype=torch.float32).reshape(-1)
        if ext.numel() != 1:
            raise RuntimeError("ContinuousConv: one extent for all points (per-point extents: use ops.continuous_conv)")
        r = ops.fixed_radius_search(inp_positions.float(), out_positions.float(), float(ext[0]) * 0.5,
                                    return_distances=False)
        out = ops.continuous_conv(self.kernel.detach(), out_positions, ext, self.offset, inp_positions, inp_features,
                                  inp_importance, r.neighbors_index, None, r.neighbors_row_splits,
                                  self.align_corners, self.coordinate_mapping, self.normalize, self.interpolation)
        if self.use_bias:
            out = out + self.bias.detach().to(out.device)
        return self.activation(out) if self.activation is not None else out
