"""ctypes binding of libo3dml_b200.so (the C ABI declared in include/o3dml_b200.h).

The argument and result types of every entry are read from the headers, which state them once for nvcc and for this
binding alike.

There is NO CPU fallback: every entry point needs the CUDA library and a CUDA
device, and fails loudly otherwise.
"""
import ctypes
import math
import os
import re

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libo3dml_b200.so")
INCLUDE = os.path.join(os.path.dirname(_HERE), "include")
_lib = None


class Src(ctypes.Structure):
    """o3dml_src_t"""
    _fields_ = [("data", ctypes.c_void_p), ("index", ctypes.c_void_p), ("rows", ctypes.c_int64),
                ("out_rows_per_batch", ctypes.c_int64), ("src_rows_per_batch", ctypes.c_int64),
                ("channels", ctypes.c_int32), ("ld", ctypes.c_int32),
                ("index_is64", ctypes.c_int32), ("index_ld", ctypes.c_int32)]


_VALUE_TYPES = {"int": ctypes.c_int, "int64_t": ctypes.c_int64, "float": ctypes.c_float, "size_t": ctypes.c_size_t,
                "unsigned long long": ctypes.c_ulonglong}
# pointers passed as plain addresses (tensor data_ptr(), host buffers, the stream)
_ADDRESS_POINTEES = {"float", "void", "int32_t", "int64_t", "int", "long long"}
_DECLARATION = re.compile(r"O3DML_API\s+([\w\s*]+?)\s*\b(\w+)\s*\(([^()]*)\)\s*;")
_PARAMETER = re.compile(r"([\w\s*]+?[\s*])(\w+)")


def _ctype(c_type, result):
    """The ctypes type of a C parameter (result=False) or return type; `const` does not matter."""
    t = re.sub(r"\s*\*", "*", " ".join(re.sub(r"\bconst\b", " ", c_type).split()))
    if t in _VALUE_TYPES:
        return _VALUE_TYPES[t]
    if t == "o3dml_src_t*":
        return ctypes.POINTER(Src)
    if t.endswith("*") and t[:-1] in _ADDRESS_POINTEES:
        return ctypes.c_void_p
    if result and t == "char*":
        return ctypes.c_char_p
    if result and t == "void":
        return None
    raise ValueError("open3d_ml_b200: no ctypes type for C %s type %r"
                     % ("return" if result else "parameter", c_type.strip()))


def declarations(header):
    """[(name, restype, argtypes)] of every `O3DML_API` prototype in a header's text, in declaration order; a name
    declared twice is listed twice.  A declaration this cannot read, or a type it has no ctypes type for, raises
    ValueError: nothing is skipped or bound to a guessed type."""
    code = re.sub(r"/\*.*?\*/|//[^\n]*", " ", header, flags=re.S)
    code = re.sub(r"^[ \t]*#.*$", "", code, flags=re.M)      # preprocessor lines, `#define O3DML_API` among them
    out = []
    for token in re.finditer(r"\bO3DML_API\b", code):
        m = _DECLARATION.match(code, token.start())
        if m is None:
            raise ValueError("open3d_ml_b200: cannot read the declaration %r" % code[token.start():].split(";")[0])
        ret, name, params = m.groups()
        args = []
        if params.strip() != "void":
            for p in params.split(","):
                pm = _PARAMETER.fullmatch(p.strip())
                if pm is None:
                    raise ValueError("open3d_ml_b200: cannot read parameter %r of %s" % (p.strip(), name))
                args.append(_ctype(pm.group(1), False))
        out.append((name, _ctype(ret, True), args))
    return out


def read_header(name):
    with open(os.path.join(INCLUDE, name)) as f:
        return f.read()


_PRODUCT_HEADER = read_header("o3dml_b200.h")
ABI_VERSION = int(re.search(r"^#define O3DML_ABI_VERSION (\d+)\s*$", _PRODUCT_HEADER, re.M).group(1))
_PRODUCT = declarations(_PRODUCT_HEADER)
EXPORTS = tuple(name for name, _, _ in _PRODUCT)           # the product ABI, in declaration order
# bring-up / profiling hooks: exported by the library and bound here, not part of the product ABI
_BRINGUP = declarations(read_header("o3dml_b200_bringup.h"))


def lib():
    """Loads (building first if the .so is absent and nvcc is available)."""
    global _lib
    if _lib is None:
        from . import build as _build
        have_nvcc = os.path.exists(_build.NVCC)
        if have_nvcc or not os.path.exists(LIB_PATH):
            # build() is a cheap mtime check when the library is current: an edited csrc/ or header is never
            # served by a stale .so; without nvcc an existing library is used as it is
            try:
                _build.build()
            except Exception as e:  # noqa: BLE001
                if not os.path.exists(LIB_PATH):
                    raise RuntimeError(
                        "open3d_ml_b200: CUDA library %s is missing and could not be built (%s). "
                        "There is no CPU fallback." % (LIB_PATH, e)) from e
                raise
        h = ctypes.CDLL(LIB_PATH)
        for name, res, args in _PRODUCT + _BRINGUP:
            fn = getattr(h, name)
            fn.restype, fn.argtypes = res, args
        if h.o3dml_abi_version() != ABI_VERSION:
            raise RuntimeError("open3d_ml_b200: ABI version mismatch")
        _lib = h
    return _lib


def check(rc):
    if rc != 0:
        raise RuntimeError("open3d_ml_b200: " + lib().o3dml_last_error().decode())


def require_cuda():
    if not torch.cuda.is_available():
        raise RuntimeError("open3d_ml_b200: no CUDA device visible; this library has no CPU path")


def ptr(t):
    return None if t is None else t.data_ptr()


def stream():
    return torch.cuda.current_stream().cuda_stream


def workspace(nbytes, device):
    """An entry point's scratch buffer: `nbytes` (its o3dml_*_workspace_bytes) of uint8 on `device`."""
    return torch.empty((nbytes,), dtype=torch.uint8, device=device)


def act_code(act):
    return {None: 0, "none": 0, "relu": 1, "leaky": 2}[act]


def is64(index):
    """The ABI's index-width flag of an int32 / int64 index tensor."""
    return 1 if index.dtype == torch.int64 else 0


def make_src(data, index=None, index_ld=1, out_rows_per_batch=0, src_rows_per_batch=0,
             channels=None, ld=None, rows=None):
    """data: 2-D float32 CUDA tensor [rows, C] (row stride ld)."""
    s = Src()
    s.data = data.data_ptr()
    s.rows = data.shape[0] if rows is None else rows
    s.channels = data.shape[1] if channels is None else channels
    s.ld = data.stride(0) if ld is None else ld
    if index is not None:
        assert index.dtype in (torch.int64, torch.int32) and index.is_cuda
        s.index = index.data_ptr()
        s.index_is64 = is64(index)
        s.index_ld = index_ld
    s.out_rows_per_batch = out_rows_per_batch
    s.src_rows_per_batch = src_rows_per_batch
    return s


def tf32_round(x):
    """fp32 -> nearest TF32 (10 explicit mantissa bits, ties to even), returned as fp32."""
    u = x.contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    u = (u + 0xFFF + ((u >> 13) & 1)) & 0xFFFFE000
    u = torch.where(u >= 2 ** 31, u - 2 ** 32, u)
    return u.to(torch.int32).view(torch.float32)


def pack_tf32_image_host(w_nk):
    """fp32 [N, K] (K contiguous) -> fp32 CPU tensor [2 * N, K]: rows [0, N) = hi = tf32(w),
    rows [N, 2N) = lo = tf32(w - hi).  gemm_tc.cu fetches [BN x 32] boxes of it by TMA."""
    w = w_nk.detach().to(torch.float32).cpu().contiguous()
    hi = tf32_round(w)
    lo = tf32_round(w - hi)
    return torch.cat([hi, lo], 0).contiguous()


def _sw128_tile(b_n32):
    """fp32 [N, 32] (one 128-byte row per output channel) -> the same tile in the K-major SWIZZLE_128B shared-memory
    layout: 16-byte chunk c of row n sits at chunk position c ^ (n & 7)."""
    n = b_n32.shape[0]
    t = b_n32.reshape(n, 8, 4)
    out = torch.empty_like(t)
    rows = torch.arange(n)
    for c in range(8):
        out[rows, c ^ (rows & 7)] = t[:, c]
    return out.reshape(n, 32)


def pack_tail_image(weights_kn, n_pads):
    """rl_tail.cu weight image: for every layer ([K, N] fp32, in x out) the TF32 hi tiles of its 32-wide k-chunks, then the
    lo tiles, each [n_pad][32] floats in the SWIZZLE_128B layout; layers concatenated."""
    parts = []
    for w, n_pad in zip(weights_kn, n_pads):
        w = w.detach().to(torch.float32).cpu()
        k, n = w.shape
        assert k % 32 == 0 and n <= n_pad
        b = torch.zeros((n_pad, k), dtype=torch.float32)
        b[:n] = w.t()
        hi = tf32_round(b)
        lo = tf32_round(b - hi)
        for img in (hi, lo):
            for c in range(k // 32):
                parts.append(_sw128_tile(img[:, 32 * c:32 * c + 32].contiguous()).reshape(-1))
    return torch.cat(parts).contiguous()


class PackedWeight:
    """A dense-layer weight in both forms: fp32 [K, Cout] for the SIMT kernel (gemm.cu) and the
    zero-padded TF32 hi/lo image [2 * n_pad, k_pad] for the wgmma kernel (gemm_tc.cu)."""

    def __init__(self, w_kc):
        w = w_kc.detach().to(torch.float32).cpu().contiguous()
        self.k, self.cout = w.shape
        self.wt = w.cuda()
        self.k_pad = (self.k + 31) // 32 * 32
        self.n_pad = 32 if self.cout <= 32 else 64 if self.cout <= 64 else (self.cout + 127) // 128 * 128
        wp = torch.zeros((self.n_pad, self.k_pad), dtype=torch.float32)
        wp[:self.cout, :self.k] = w.t()
        self.img = pack_tf32_image_host(wp).cuda()
        self.host = w                      # fp32 [K, Cout] on the host: rowmlp.cu takes it by value
        self._host_affine = {}

    def host_affine(self, scale, shift):
        """Host copies of the folded-BN scale / shift of this layer (made once, at first use).  The cache
        entry keeps the device tensors alive (so their addresses cannot be reused by other tensors) and is
        keyed by their version counters (an in-place update invalidates it)."""
        def k(t):
            return (0, 0) if t is None else (t.data_ptr(), t._version)
        key = (k(scale), k(shift))
        ent = self._host_affine.get(key)
        if ent is None:
            ent = (None if scale is None else scale.detach().float().cpu().contiguous(),
                   None if shift is None else shift.detach().float().cpu().contiguous(), scale, shift)
            if len(self._host_affine) > 8:      # a layer has one (scale, shift) pair; do not grow without bound
                self._host_affine.clear()
            self._host_affine[key] = ent
        return ent[0], ent[1]

    @property
    def shape(self):
        return (self.k, self.cout)


def pack_linear(w_kc):
    return PackedWeight(w_kc)


def host_state_dict(state_dict):
    """A reference state_dict on the host: floating-point entries as fp32 copies, the others as they are."""
    return {k: v.detach().to("cpu", torch.float32) if v.is_floating_point() else v.cpu()
            for k, v in state_dict.items()}


def fold_bn(sd, prefix, eps, bias=None):
    """Eval-mode BatchNorm `prefix` after a layer with an optional `bias`, folded in float64 into fp32 (scale, shift):
    s = w / sqrt(var + eps), t = b - s * mean [+ s * bias]."""
    s = sd[prefix + ".weight"].double() / torch.sqrt(sd[prefix + ".running_var"].double() + eps)
    t = sd[prefix + ".bias"].double() - s * sd[prefix + ".running_mean"].double()
    if bias is not None:
        t = t + s * bias.double()
    return s.float(), t.float()


TC_MIN_K = 64


def _tc_ok(srcs):
    """Tensor-core kernel only where it pays (K >= TC_MIN_K) and where the operand contract of gemm_tc.cu
    holds: every source 4-channel aligned with 16-byte aligned rows, and every source but the last a
    multiple of 32 channels (a 32-channel k-slice never straddles two sources)."""
    if sum(s.channels for s in srcs) < TC_MIN_K:
        return False
    if any(s.channels % 32 for s in srcs[:-1]):
        return False
    return all((s.channels % 4 == 0) and (s.ld % 4 == 0) and (s.data % 16 == 0) for s in srcs)


USE_ROW_MLP = True
# one-thread-per-row layers need rows >= SMs x 256 x a few to fill the machine: below this the tensor-core kernel
# (128 rows per CTA, K >= TC_MIN_K) has the shorter critical path
ROW_MLP_MIN_ROWS = 40000


def _rows_small_ok(srcs, out, ld, co):
    """Alignment contract of rowmlp.cu: float4 access wherever a width is a multiple of 4."""
    for s in srcs:
        if s.channels % 4 == 0 and (s.ld % 4 or s.data % 16):
            return False
    return not (co % 4 == 0 and (ld % 4 or out.data_ptr() % 16))


def linear(srcs, weight, out, scale=None, shift=None, residual=None, act=None, slope=0.0,
           num_rows=None, out_channels=None, out_ld=None, out_nchw_plane=0):
    """out[n,:] = act(scale * (concat(srcs)[n] @ W) + shift + residual[n]).  `weight` is either an
    fp32 [K, Cout] tensor (SIMT kernel) or a PackedWeight (tensor-core kernel when the sources
    allow it)."""
    arr = (Src * len(srcs))(*srcs)
    n = out.shape[0] if num_rows is None else num_rows
    packed = isinstance(weight, PackedWeight)
    wt = weight.wt if packed else weight
    co = wt.shape[1] if out_channels is None else out_channels
    ld = (out.stride(0) if out_nchw_plane == 0 else co) if out_ld is None else out_ld
    res_ld = residual.stride(0) if residual is not None else 0
    prefer_tc = packed and n < ROW_MLP_MIN_ROWS and _tc_ok(srcs)
    if (packed and USE_ROW_MLP and not prefer_tc and residual is None and out_nchw_plane == 0 and len(srcs) <= 2 and
            lib().o3dml_linear_rows_small_supported(srcs[0].channels, srcs[1].channels if len(srcs) == 2 else 0,
                                                    co) and _rows_small_ok(srcs, out, ld, co)):
        hs, ht = weight.host_affine(scale, shift)
        check(lib().o3dml_linear_rows_small(n, arr, len(srcs), weight.host.data_ptr(), ptr(hs), ptr(ht),
                                            act_code(act), float(slope), ptr(out), ld, co, stream()))
    elif packed and _tc_ok(srcs):
        check(lib().o3dml_linear_tc(n, arr, len(srcs), ptr(weight.img), weight.k_pad, weight.n_pad,
                                    ptr(scale), ptr(shift), ptr(residual), res_ld, act_code(act),
                                    float(slope), ptr(out), ld, co, out_nchw_plane, stream()))
    else:
        check(lib().o3dml_linear(n, arr, len(srcs), ptr(wt), ptr(scale), ptr(shift), ptr(residual),
                                 res_ld, act_code(act), float(slope), ptr(out), ld, co, out_nchw_plane,
                                 stream()))
    return out


def conv3x3(x, weight, out, scale=None, shift=None, stride=1, act=None, slope=0.0):
    """out = act(scale * conv3x3(x) + shift): padding 1, stride 1 or 2, x [B, H, W, C] and out [B, OH, OW, Cout]
    contiguous NHWC.  `weight` [9 C, Cout] (row (ky * 3 + kx) * C + c) is either an fp32 tensor (SIMT kernel) or a
    PackedWeight (tensor-core kernel when C % 32 == 0, SIMT otherwise)."""
    B, H, W, C = x.shape
    co = out.shape[3]
    if isinstance(weight, PackedWeight) and C % 32 == 0:
        check(lib().o3dml_conv3x3_nhwc_tc(ptr(x), B, H, W, C, stride, ptr(weight.img), weight.k_pad, weight.n_pad,
                                          ptr(scale), ptr(shift), act_code(act), float(slope), ptr(out), co, stream()))
    else:
        wt = weight.wt if isinstance(weight, PackedWeight) else weight
        check(lib().o3dml_conv3x3_nhwc(ptr(x), B, H, W, C, stride, ptr(wt), ptr(scale), ptr(shift), act_code(act),
                                       float(slope), ptr(out), co, stream()))
    return out


def conv3x3x3(x, weight, out, scale=None, shift=None, act=None, slope=0.0):
    """out = act(scale * conv3x3x3(x) + shift): padding 1, stride 1, x [B, X, Y, Z, C] and out [B, X, Y, Z, Cout]
    contiguous channels-last grids, C % 32 == 0.  `weight` is the PackedWeight of [27 C, Cout], row
    ((kx * 3 + ky) * 3 + kz) * C + c.  There is one kernel, on the tensor cores."""
    B, X, Y, Z, C = x.shape
    check(lib().o3dml_conv3x3x3_ndhwc_tc(ptr(x), B, X, Y, Z, C, ptr(weight.img), weight.k_pad, weight.n_pad,
                                         ptr(scale), ptr(shift), act_code(act), float(slope), ptr(out), out.shape[4],
                                         stream()))
    return out


def deconv(x, weight, out, scale=None, shift=None, stride=1, act=None, slope=0.0):
    """ConvTranspose2d with kernel == stride: out = act(scale * deconv(x) + shift), x [B, H, W, C] contiguous NHWC,
    out [B, H * stride, W * stride, Cout] NHWC with unit channel stride, possibly a channel slice of a wider buffer.
    `weight` [C, stride^2 * Cout] (column (ky * stride + kx) * Cout + co); scale / shift tiled to [stride^2 * Cout].
    An fp32 tensor runs the SIMT kernel; a PackedWeight the tensor-core kernel when C % 4 == 0, SIMT otherwise."""
    B, H, W, C = x.shape
    co, ld = out.shape[3], out.stride(2)
    if out.stride(3) != 1 or out.stride(1) != out.shape[2] * ld or out.stride(0) != out.shape[1] * out.stride(1):
        raise ValueError("deconv: out must be NHWC rows of a uniform stride")
    if isinstance(weight, PackedWeight) and C % 4 == 0:
        check(lib().o3dml_deconv_nhwc_tc(ptr(x), B, H, W, C, stride, ptr(weight.img), weight.k_pad, weight.n_pad,
                                         ptr(scale), ptr(shift), act_code(act), float(slope), ptr(out), ld, co,
                                         stream()))
    else:
        wt = weight.wt if isinstance(weight, PackedWeight) else weight
        check(lib().o3dml_deconv_nhwc(ptr(x), B, H, W, C, stride, ptr(wt), ptr(scale), ptr(shift), act_code(act),
                                      float(slope), ptr(out), ld, co, stream()))
    return out


def pack_operand_image_host(w_nk):
    """fp32 [N, K] (K contiguous, i.e. nn.Linear's [out, in]) -> uint8 CPU tensor holding the
    3xFP16 operand images of csrc/tc.cuh: [K/8][N][8 halves] of hi = fp16(w), then the same
    layout of lo = fp16(w - hi).  Like the kernels' split (tc.cuh split8), nothing is clamped: a weight of magnitude
    >= 65520, Inf or NaN gives a non-finite hi or lo, so the product it enters is non-finite rather than silently wrong."""
    w = w_nk.detach().to(torch.float32).cpu()
    n, k = w.shape
    assert k % 8 == 0 and n % 8 == 0
    hi = w.to(torch.float16)
    lo = (w - hi.to(torch.float32)).to(torch.float16)

    def img(h):
        return h.view(n, k // 8, 8).permute(1, 0, 2).contiguous().view(-1)
    return torch.cat([img(hi), img(lo)]).view(torch.uint8)


def pack_operand_image(w_nk):
    """pack_operand_image_host, moved to the device."""
    return pack_operand_image_host(w_nk).cuda()


def pack_lfa16_weights(w10_t, s10, t10, wl2_t, s2, t2, wscore_t, bscore):
    """The host weight block of o3dml_randla_lfa16_pool (O3DML_LFA16_WEIGHT_FLOATS = 448 floats): w10_t [10, 8], s10,
    t10 [8], wl2_t [8, 8], s2, t2 [8], wscore_t [16, 16], bscore [16], matrices [in, out], concatenated in that order.
    Returns a float32 CPU tensor."""
    parts = [t.detach().to("cpu", torch.float32).reshape(-1) for t in (w10_t, s10, t10, wl2_t, s2, t2, wscore_t, bscore)]
    assert [p.numel() for p in parts] == [80, 8, 8, 64, 8, 8, 256, 16], [p.numel() for p in parts]
    return torch.cat(parts).contiguous()
