"""Torch-tensor front end of the C ABI (``include/slowfast_b200.h``).

PyTorch is used for device memory, streams and dtype bookkeeping only; every function here enqueues one or more
of the library's own kernels on the current CUDA stream.  There is no CPU path: without the native library or a
CUDA device the calls raise ``NativeLibraryError``.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Optional, Sequence, Tuple

import torch

from . import lib as L

BF16 = torch.bfloat16
F32 = torch.float32

# launch counter: bench.py reports how many of OUR kernels launches were enqueued inside the timed region
_launches = 0


def launches() -> int:
    return _launches


def _count(n: int = 1) -> None:
    global _launches
    _launches += n


def add_launches(n: int) -> None:
    """Account for kernel launches replayed from a captured CUDA graph."""
    _count(n)


def _stream() -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def pad8(c: int) -> int:
    return (c + 7) // 8 * 8


@dataclass
class Planes:
    """Split-bf16 activation, channels-last [n, t, h, w, c] view into storage with channel pitch ``pitch``.

    ``hi``/``lo`` are the *storage* tensors ([n,t,h,w,pitch] bf16); ``c0`` is the first channel of the view.
    ``lo`` is None in fast (bf16) mode."""

    hi: torch.Tensor
    lo: Optional[torch.Tensor]
    n: int
    t: int
    h: int
    w: int
    c: int
    c0: int = 0

    @property
    def pitch(self) -> int:
        return self.hi.shape[-1]

    @property
    def rows(self) -> int:
        return self.n * self.t * self.h * self.w

    def hi_ptr(self) -> int:
        return self.hi.data_ptr() + 2 * self.c0

    def lo_ptr(self) -> Optional[int]:
        return None if self.lo is None else self.lo.data_ptr() + 2 * self.c0

    def slice(self, c0: int, c: int) -> "Planes":
        assert c0 % 8 == 0 and c % 8 == 0 and c0 + c <= self.c
        return Planes(self.hi, self.lo, self.n, self.t, self.h, self.w, c, self.c0 + c0)

    def to_float(self) -> torch.Tensor:
        """Reconstruct fp32 values of the view (debug / tests)."""
        x = self.hi[..., self.c0:self.c0 + self.c].float()
        if self.lo is not None:
            x = x + self.lo[..., self.c0:self.c0 + self.c].float()
        return x


def alloc_planes(n, t, h, w, c, nsplit: int, device, pitch: Optional[int] = None) -> Planes:
    pitch = pitch or c
    hi = torch.empty((n, t, h, w, pitch), dtype=BF16, device=device)
    lo = torch.empty((n, t, h, w, pitch), dtype=BF16, device=device) if nsplit == 3 else None
    return Planes(hi, lo, n, t, h, w, c, 0)


@dataclass
class F32View:
    """fp32 [rows, c] matrix view with a row pitch (channel slice of a wider channels-last tensor)."""

    t: torch.Tensor  # storage
    rows: int
    c: int
    pitch: int
    c0: int = 0

    def ptr(self) -> int:
        return self.t.data_ptr() + 4 * self.c0

    def as_tensor(self) -> torch.Tensor:
        return self.t.reshape(self.rows, self.pitch)[:, self.c0:self.c0 + self.c]


def f32view(t: torch.Tensor, c: Optional[int] = None, c0: int = 0) -> F32View:
    pitch = t.shape[-1]
    return F32View(t, t.numel() // pitch, c if c is not None else pitch, pitch, c0)


def zero_f32(v: "F32View") -> None:
    lib = L.load()
    L.check(lib.sfb_zero_f32_2d(v.ptr(), v.rows, v.c, v.pitch, _stream()), "sfb_zero_f32_2d")
    _count()


def add_f32(dst: "F32View", src: "F32View") -> None:
    lib = L.load()
    assert dst.rows == src.rows and dst.c == src.c
    L.check(lib.sfb_add_f32_2d(dst.ptr(), src.ptr(), dst.rows, dst.c, dst.pitch, src.pitch, _stream()),
            "sfb_add_f32_2d")
    _count()


# ------------------------------------------------------------------------------------------------ packing
def split_planes(x: torch.Tensor, out: Planes) -> None:
    """fp32 channels-last tensor [..., c] -> planes."""
    lib = L.load()
    assert x.dtype == F32 and x.is_contiguous() and x.shape[-1] == out.c
    L.check(lib.sfb_split_planes(x.data_ptr(), out.rows, out.c, x.shape[-1], out.hi_ptr(), out.lo_ptr(), out.pitch,
                                 _stream()), "sfb_split_planes")
    _count()


def input_pack(x: torch.Tensor, out: Planes) -> None:
    """NCDHW fp32 clip -> NDHWC planes padded to out.c channels."""
    lib = L.load()
    n, c, t, h, w = x.shape
    assert x.dtype == F32 and x.is_contiguous() and out.pitch == out.c and out.c0 == 0
    L.check(lib.sfb_input_pack(x.data_ptr(), n, c, t, h, w, out.c, out.hi_ptr(), out.lo_ptr(), _stream()),
            "sfb_input_pack")
    _count()


@dataclass
class FilterMat:
    """GEMM filter matrix planes [rows, ntaps * cols_pad]."""

    hi: torch.Tensor
    lo: Optional[torch.Tensor]
    rows: int
    ntaps: int
    cols_pad: int


def filter_pack(w: torch.Tensor, out: FilterMat, tapmap: Optional[Sequence[int]] = None,
                transpose: bool = False) -> None:
    lib = L.load()
    assert w.dtype == F32 and w.is_contiguous()
    cout, cin = w.shape[0], w.shape[1]
    taps_total = w[0, 0].numel() if w.dim() > 2 else 1
    ntaps = out.ntaps
    tm = None
    if tapmap is not None:
        assert len(tapmap) == ntaps
        tm = (C.c_int32 * ntaps)(*tapmap)
    L.check(lib.sfb_filter_pack(w.data_ptr(), cout, cin, taps_total, tm, ntaps, 1 if transpose else 0, out.cols_pad,
                                out.hi.data_ptr(), _ptr(out.lo), _stream()), "sfb_filter_pack")
    _count()


def alloc_filter(rows: int, ntaps: int, cols: int, nsplit: int, device) -> FilterMat:
    cp = pad8(cols)
    hi = torch.empty((rows, ntaps * cp), dtype=BF16, device=device)
    lo = torch.empty((rows, ntaps * cp), dtype=BF16, device=device) if nsplit == 3 else None
    return FilterMat(hi, lo, rows, ntaps, cp)


def filter_unpack_grad(dwm: torch.Tensor, dw: torch.Tensor, cin_pad: int, accumulate: bool) -> None:
    lib = L.load()
    cout, cin = dw.shape[0], dw.shape[1]
    taps = dw[0, 0].numel() if dw.dim() > 2 else 1
    assert dw.is_contiguous() and dwm.is_contiguous()
    L.check(lib.sfb_filter_unpack_grad(dwm.data_ptr(), dw.data_ptr(), cout, cin, taps, cin_pad,
                                       1 if accumulate else 0, _stream()), "sfb_filter_unpack_grad")
    _count()


# ------------------------------------------------------------------------------------------------ convolution
@dataclass
class ConvGeom:
    """Geometry of one implicit-GEMM problem: taps, dilation, traversal stride, lower corner and output grid."""

    k: Tuple[int, int, int]
    stride: Tuple[int, int, int] = (1, 1, 1)
    low: Tuple[int, int, int] = (0, 0, 0)
    out: Tuple[int, int, int] = (1, 1, 1)
    dil: Tuple[int, int, int] = (1, 1, 1)


def conv_out_size(i: int, k: int, s: int, p: int, d: int = 1) -> int:
    return (i + 2 * p - d * (k - 1) - 1) // s + 1


def fprop_geom(x: Planes, k, stride, pad, dil=(1, 1, 1)) -> ConvGeom:
    out = tuple(conv_out_size(i, kk, s, p, d) for i, kk, s, p, d in zip((x.t, x.h, x.w), k, stride, pad, dil))
    return ConvGeom(tuple(k), tuple(stride), tuple(-p for p in pad), out, tuple(dil))


def conv_m_tiles(n: int, geom: ConvGeom) -> int:
    m = n * geom.out[0] * geom.out[1] * geom.out[2]
    return (m + 127) // 128


def conv_igemm(x: Planes, f: FilterMat, geom: ConvGeom, out: torch.Tensor, out_strides: Tuple[int, int, int, int],
               out_offset: int = 0, accumulate: bool = False, stats: Optional[torch.Tensor] = None,
               nsplit: int = 3) -> None:
    """out view[n, z, p, q, :f.rows] (+)= conv(x, f).  ``out_strides`` are element strides for (n, t, h, w);
    ``out_offset`` an element offset into ``out`` (channel slice / strided scatter)."""
    lib = L.load()
    assert f.cols_pad == x.c, (f.cols_pad, x.c)
    d = L.ConvDesc()
    d.a_hi, d.a_lo = x.hi_ptr(), x.lo_ptr()
    d.n, d.d, d.h, d.w, d.c, d.c_pitch = x.n, x.t, x.h, x.w, x.c, x.pitch
    d.b_hi, d.b_lo = f.hi.data_ptr(), _ptr(f.lo)
    d.cout = f.rows
    d.kt, d.kh, d.kw = geom.k
    d.dil_t, d.dil_h, d.dil_w = geom.dil
    d.str_t, d.str_h, d.str_w = geom.stride
    d.low_t, d.low_h, d.low_w = geom.low
    d.out_t, d.out_h, d.out_w = geom.out
    d.out = out.data_ptr() + 4 * out_offset
    d.os_n, d.os_t, d.os_h, d.os_w = out_strides
    d.accumulate = int(accumulate)     # 0 overwrite, 1 read-modify-write, 2 fire-and-forget float atomics (same sums)
    d.stats = _ptr(stats)
    d.nsplit = nsplit
    L.check(lib.sfb_conv_igemm(C.byref(d), _stream()), "sfb_conv_igemm")
    _count()


def conv_wgrad(x: Planes, dy: Planes, geom: ConvGeom, dwm: torch.Tensor, nsplit: int = 3) -> None:
    """dwm[cout, taps*x.c] += dY^T * im2col(x).  dy must be dense rows [M, cout] (its pitch may exceed cout)."""
    lib = L.load()
    d = L.WgradDesc()
    d.x_hi, d.x_lo = x.hi_ptr(), x.lo_ptr()
    d.n, d.d, d.h, d.w, d.c, d.c_pitch = x.n, x.t, x.h, x.w, x.c, x.pitch
    d.dy_hi, d.dy_lo = dy.hi_ptr(), dy.lo_ptr()
    d.cout, d.dy_pitch = dy.c, dy.pitch
    d.kt, d.kh, d.kw = geom.k
    d.dil_t, d.dil_h, d.dil_w = geom.dil
    d.str_t, d.str_h, d.str_w = geom.stride
    d.low_t, d.low_h, d.low_w = geom.low
    d.out_t, d.out_h, d.out_w = geom.out
    assert dy.rows == x.n * geom.out[0] * geom.out[1] * geom.out[2]
    d.dw = dwm.data_ptr()
    d.nsplit = nsplit
    L.check(lib.sfb_conv_wgrad(C.byref(d), _stream()), "sfb_conv_wgrad")
    _count()


# ------------------------------------------------------------------------------------------------ batch norm
def bn_finalize(partials: Optional[torch.Tensor], m_tiles: int, c: int, count: int, gamma, beta, running_mean,
                running_var, momentum: float, eps: float, training: bool, scale, shift, save_mean, save_invstd):
    lib = L.load()
    L.check(lib.sfb_bn_finalize(_ptr(partials), m_tiles, c, count, _ptr(gamma), _ptr(beta), _ptr(running_mean),
                                _ptr(running_var), momentum, eps, 1 if training else 0, scale.data_ptr(),
                                shift.data_ptr(), _ptr(save_mean), _ptr(save_invstd), _stream()), "sfb_bn_finalize")
    _count()


def bn_apply(y: F32View, scale, shift, out: Planes, relu: bool, y2: Optional[F32View] = None, scale2=None,
             shift2=None, res: Optional[Planes] = None) -> None:
    lib = L.load()
    d = L.BnApplyDesc()
    d.y, d.y_pitch, d.scale, d.shift = y.ptr(), y.pitch, scale.data_ptr(), shift.data_ptr()
    if y2 is not None:
        d.y2, d.y2_pitch, d.scale2, d.shift2 = y2.ptr(), y2.pitch, scale2.data_ptr(), shift2.data_ptr()
    if res is not None:
        assert res.c == out.c and res.rows == out.rows
        d.res_hi, d.res_lo, d.res_pitch = res.hi_ptr(), res.lo_ptr(), res.pitch
    d.out_hi, d.out_lo, d.out_pitch = out.hi_ptr(), out.lo_ptr(), out.pitch
    d.rows, d.c, d.relu = out.rows, out.c, 1 if relu else 0
    assert y.rows == out.rows and y.c == out.c
    L.check(lib.sfb_bn_apply(C.byref(d), _stream()), "sfb_bn_apply")
    _count()


def bn_bwd_scratch(rows: int, c: int, device):
    lib = L.load()
    nb = lib.sfb_bn_bwd_blocks(rows, c)
    return (torch.empty((nb, 2, c), dtype=F32, device=device), torch.empty((3, c), dtype=F32, device=device))


def bn_bwd(dout: F32View, mask: Optional[Planes], y: F32View, mean, invstd, gamma, dgamma, dbeta, dy: Planes,
           partials, coef, training: bool = True, accumulate_param_grads: bool = False,
           dres: Optional[F32View] = None, dres_accumulate: bool = False, c_valid: int = 0,
           mask_affine=None) -> None:
    """``mask``: post-ReLU planes (ReLU mask = planes > 0) or None; ``mask_affine`` = (scale, shift): recompute the
    mask as y*scale + shift > 0 instead (used when the activation was never materialised)."""
    lib = L.load()
    d = L.BnBwdDesc()
    d.c_valid = c_valid
    if mask_affine is not None:
        assert mask is None
        d.mask_scale, d.mask_shift = mask_affine[0].data_ptr(), mask_affine[1].data_ptr()
    d.dout, d.dout_pitch = dout.ptr(), dout.pitch
    if mask is not None:
        d.mask_hi, d.mask_pitch = mask.hi_ptr(), mask.pitch
    d.y, d.y_pitch = y.ptr(), y.pitch
    d.mean, d.invstd, d.gamma = mean.data_ptr(), invstd.data_ptr(), _ptr(gamma)
    d.dgamma, d.dbeta = _ptr(dgamma), _ptr(dbeta)
    d.accumulate_param_grads = 1 if accumulate_param_grads else 0
    d.training = 1 if training else 0
    d.dy_hi, d.dy_lo, d.dy_pitch = dy.hi_ptr(), dy.lo_ptr(), dy.pitch
    if dres is not None:
        d.dres, d.dres_pitch, d.dres_accumulate = dres.ptr(), dres.pitch, 1 if dres_accumulate else 0
    d.partials, d.coef = partials.data_ptr(), coef.data_ptr()
    d.rows, d.c = dy.rows, dy.c
    assert dout.rows == dy.rows and y.rows == dy.rows
    L.check(lib.sfb_bn_bwd(C.byref(d), _stream()), "sfb_bn_bwd")
    _count(3)


def _pool_desc(n, t, h, w, c, oh, ow, k, s, p):
    d = L.PoolDesc()
    d.n, d.t, d.h, d.w, d.c, d.oh, d.ow = n, t, h, w, c, oh, ow
    d.kh, d.kw = k
    d.sh, d.sw = s
    d.ph, d.pw = p
    return d


def bn_relu_maxpool_fwd(y: torch.Tensor, scale, shift, out: Planes, argmax: torch.Tensor, k, s, p) -> None:
    lib = L.load()
    n, t, h, w, c = y.shape
    d = _pool_desc(n, t, h, w, c, out.h, out.w, k, s, p)
    d.y, d.scale, d.shift = y.data_ptr(), scale.data_ptr(), shift.data_ptr()
    d.out_hi, d.out_lo, d.out_pitch = out.hi_ptr(), out.lo_ptr(), out.pitch
    d.argmax = argmax.data_ptr()
    L.check(lib.sfb_bn_relu_maxpool_fwd(C.byref(d), _stream()), "sfb_bn_relu_maxpool_fwd")
    _count()


def bn_relu_maxpool_bwd(dout: F32View, argmax: torch.Tensor, dz: torch.Tensor, oh, ow, k, s, p) -> None:
    lib = L.load()
    n, t, h, w, c = dz.shape
    d = _pool_desc(n, t, h, w, c, oh, ow, k, s, p)
    d.argmax = argmax.data_ptr()
    d.dout, d.dout_pitch = dout.ptr(), dout.pitch
    d.dz = dz.data_ptr()
    L.check(lib.sfb_bn_relu_maxpool_bwd(C.byref(d), _stream()), "sfb_bn_relu_maxpool_bwd")
    _count()


# ------------------------------------------------------------------------------------------------ head
def global_avgpool_fwd(x: Planes, out: torch.Tensor, col0: int = 0) -> None:
    """out[n, col0:col0+c] = mean over (t,h,w) of x."""
    lib = L.load()
    assert out.dtype == F32 and out.dim() == 2 and out.is_contiguous()
    L.check(lib.sfb_global_avgpool_fwd(x.hi_ptr(), x.lo_ptr(), x.pitch, x.n, x.t * x.h * x.w, x.c,
                                       out.data_ptr() + 4 * col0, out.shape[1], _stream()), "sfb_global_avgpool_fwd")
    _count()


def global_avgpool_bwd(dpooled: torch.Tensor, col0: int, n: int, spatial: int, c: int, dx: F32View) -> None:
    lib = L.load()
    L.check(lib.sfb_global_avgpool_bwd(dpooled.data_ptr() + 4 * col0, dpooled.shape[1], n, spatial, c, dx.ptr(),
                                       dx.pitch, _stream()), "sfb_global_avgpool_bwd")
    _count()


def window_avgpool_fwd(x: Planes, k: Tuple[int, int, int], out: torch.Tensor, col0: int = 0) -> None:
    """out[(n,z,p,q), col0:col0+c] = mean of the stride-1 window k of x (AvgPool3d(k, stride=1))."""
    lib = L.load()
    assert out.dtype == F32 and out.dim() == 2 and out.is_contiguous()
    L.check(lib.sfb_window_avgpool_fwd(x.hi_ptr(), x.lo_ptr(), x.pitch, x.n, x.t, x.h, x.w, x.c, k[0], k[1], k[2],
                                       out.data_ptr() + 4 * col0, out.shape[1], _stream()), "sfb_window_avgpool_fwd")
    _count()


def rows_group_mean(x: torch.Tensor, out: torch.Tensor, g: int) -> None:
    lib = L.load()
    n, k = out.shape
    assert x.shape == (n * g, k) and x.is_contiguous() and out.is_contiguous()
    L.check(lib.sfb_rows_group_mean(x.data_ptr(), out.data_ptr(), n, g, k, _stream()), "sfb_rows_group_mean")
    _count()


def dropout_fwd(x: torch.Tensor, mask: torch.Tensor, p: float, seed: int,
                step: Optional[torch.Tensor] = None) -> None:
    """``step``: optional int64 device counter mixed into the seed and incremented after use (graph-replay safe)."""
    lib = L.load()
    L.check(lib.sfb_dropout_fwd(x.data_ptr(), mask.data_ptr(), x.numel(), p, seed & (2 ** 64 - 1), _ptr(step),
                                _stream()), "sfb_dropout_fwd")
    _count(2 if step is not None else 1)


def dropout_bwd(dx: torch.Tensor, mask: torch.Tensor, p: float) -> None:
    lib = L.load()
    L.check(lib.sfb_dropout_bwd(dx.data_ptr(), mask.data_ptr(), dx.numel(), p, _stream()), "sfb_dropout_bwd")
    _count()


def small_linear_fwd(x, w, b, y) -> None:
    lib = L.load()
    m, j = x.shape
    k = w.shape[0]
    L.check(lib.sfb_small_linear_fwd(x.data_ptr(), w.data_ptr(), _ptr(b), y.data_ptr(), m, k, j, _stream()),
            "sfb_small_linear_fwd")
    _count()


def small_linear_bwd(dy, x, w, dw, db, dx, accumulate: bool = False) -> None:
    lib = L.load()
    m, j = x.shape
    k = w.shape[0]
    L.check(lib.sfb_small_linear_bwd(dy.data_ptr(), x.data_ptr(), w.data_ptr(), _ptr(dw), _ptr(db), _ptr(dx), m, k, j,
                                     1 if accumulate else 0, _stream()), "sfb_small_linear_bwd")
    _count((1 if dw is not None else 0) + (1 if dx is not None else 0))


def row_softmax(x: torch.Tensor) -> None:
    lib = L.load()
    L.check(lib.sfb_row_softmax(x.data_ptr(), x.shape[0], x.shape[1], _stream()), "sfb_row_softmax")
    _count()


# ------------------------------------------------------------------------------------------------ stem (W-shift)
@dataclass
class StemGeom:
    """Folded geometry of a C_in<=4, W-stride-2 stem conv (see csrc/conv_stem.cu)."""

    cin: int
    cout: int
    k: Tuple[int, int, int]       # original (kt, kh, kw)
    stride: Tuple[int, int, int]  # original; stride[2] must be 2
    pad: Tuple[int, int, int]

    @property
    def dmin(self) -> int:
        return -((self.pad[2] + 1) // 2)  # floor(-pad_w / 2)

    @property
    def kwf(self) -> int:
        return (self.k[2] - 1 - self.pad[2]) // 2 - self.dmin + 1

    @property
    def pad_wf(self) -> int:
        return -self.dmin

    @property
    def kfold(self) -> int:
        return self.k[0] * self.k[1] * self.kwf * 8

    def out_dims(self, t, h, w):
        return tuple(conv_out_size(i, kk, s, p) for i, kk, s, p in zip((t, h, w), self.k, self.stride, self.pad))


def stem_supported(cin, k, stride, pad, w) -> bool:
    g = StemGeom(cin, 8, tuple(k), tuple(stride), tuple(pad))
    return cin <= 4 and stride[2] == 2 and w % 2 == 0 and g.kwf in (2, 4) and conv_out_size(w, k[2], 2, pad[2]) == w // 2


def stem_input_fold(x: torch.Tensor, out: Planes) -> None:
    lib = L.load()
    n, c, t, h, w = x.shape
    assert out.c == 8 and out.pitch == 8 and out.w == w // 2 and x.is_contiguous() and x.dtype == F32
    L.check(lib.sfb_stem_input_fold(x.data_ptr(), n, c, t, h, w, out.hi_ptr(), out.lo_ptr(), _stream()),
            "sfb_stem_input_fold")
    _count()


def stem_filter_fold(w: torch.Tensor, g: StemGeom, f: FilterMat) -> None:
    lib = L.load()
    L.check(lib.sfb_stem_filter_fold(w.data_ptr(), None, g.cout, g.cin, g.k[0], g.k[1], g.k[2], g.pad[2], g.kwf,
                                     f.hi.data_ptr(), _ptr(f.lo), None, 0, _stream()), "sfb_stem_filter_fold")
    _count()


def stem_filter_unfold_grad(gmat: torch.Tensor, dw: torch.Tensor, g: StemGeom) -> None:
    lib = L.load()
    L.check(lib.sfb_stem_filter_fold(None, dw.data_ptr(), g.cout, g.cin, g.k[0], g.k[1], g.k[2], g.pad[2], g.kwf,
                                     None, None, gmat.data_ptr(), 1, _stream()), "sfb_stem_filter_fold(reverse)")
    _count()


def _stem_desc(x: Planes, g: StemGeom, nsplit: int):
    d = L.StemDesc()
    d.x_hi, d.x_lo = x.hi_ptr(), x.lo_ptr()
    d.n, d.t, d.h, d.wf = x.n, x.t, x.h, x.w
    d.cout, d.kt, d.kh, d.kwf = g.cout, g.k[0], g.k[1], g.kwf
    d.str_t, d.str_h = g.stride[0], g.stride[1]
    d.pad_t, d.pad_h, d.pad_wf = g.pad[0], g.pad[1], g.pad_wf
    d.out_t, d.out_h, d.out_w = g.out_dims(x.t, x.h, 2 * x.w)
    d.nsplit = nsplit
    return d


def stem_m_tiles(x: Planes, g: StemGeom) -> int:
    return int(L.load().sfb_stem_m_tiles(C.byref(_stem_desc(x, g, 1))))


def stem_fprop(x: Planes, f: FilterMat, g: StemGeom, out: torch.Tensor, stats: Optional[torch.Tensor],
               nsplit: int = 3) -> None:
    """W-shift stem forward (csrc/conv_stem.cu): up to 128 output channels (one accumulator tile of 128 columns); the
    stems of the supported models have 8, 24 or 64."""
    lib = L.load()
    d = _stem_desc(x, g, nsplit)
    d.f_hi, d.f_lo = f.hi.data_ptr(), _ptr(f.lo)
    d.out, d.stats = out.data_ptr(), _ptr(stats)
    L.check(lib.sfb_stem_fprop(C.byref(d), _stream()), "sfb_stem_fprop")
    _count()


def stem_wgrad(x: Planes, dy: Planes, g: StemGeom, dwm: torch.Tensor, nsplit: int = 3) -> None:
    """W-shift stem weight gradient (csrc/conv_stem.cu): up to 64 output channels and 4 folded W taps (filters up to 7
    wide at stride 2)."""
    lib = L.load()
    assert dy.pitch == dy.c == g.cout
    d = _stem_desc(x, g, nsplit)
    d.dy_hi, d.dy_lo = dy.hi_ptr(), dy.lo_ptr()
    d.dwm = dwm.data_ptr()
    L.check(lib.sfb_stem_wgrad(C.byref(d), _stream()), "sfb_stem_wgrad")
    _count()


# ------------------------------------------------------------------------------------------------ stem (Toeplitz, cout = 8)
def stem8_mr(w: int) -> int:
    """Granule rows per folded input row (and per operand array): OW/8 groups of 8 output pixels + one halo row."""
    return w // 16 + 1


def stem8_plane_dims(n, t, h, w):
    """Storage dims of the de-interleaved folded clip: [n][2t + (h & 1)][h/2][(j, m) = 8 * MR granules][8 slots]."""
    return n, 2 * t, h // 2, 8 * stem8_mr(w), 8


def _stem8_desc(x: Planes, g: StemGeom, nsplit: int):
    d = L.StemDesc()
    d.x_hi, d.x_lo = x.hi_ptr(), x.lo_ptr()
    t, h, w = x.t // 2, x.h * 2, (x.w // 8 - 1) * 16
    d.n, d.t, d.h, d.wf = x.n, t, h, x.w
    d.cout, d.kt, d.kh, d.kwf = g.cout, g.k[0], g.k[1], g.kwf
    d.str_t, d.str_h = g.stride[0], g.stride[1]
    d.pad_t, d.pad_h, d.pad_wf = g.pad[0], g.pad[1], g.pad_wf
    d.out_t, d.out_h, d.out_w = g.out_dims(t, h, w)
    d.nsplit = nsplit
    return d


def stem8_supported(cin, cout, k, stride, pad, t, h, w) -> bool:
    """Geometry test of the Toeplitz stem kernels (csrc/conv_stem8.cu): 3 -> 8 channels, [kt,7,7], stride (1,2,2), pad 3."""
    if not (cin <= 4 and cout == 8 and tuple(k[1:]) == (7, 7) and tuple(stride) == (1, 2, 2) and tuple(pad[1:]) == (3, 3)
            and w % 16 == 0 and h % 16 == 0 and w <= 240 and 1 <= k[0] <= 8):
        return False
    g = StemGeom(cin, cout, tuple(k), tuple(stride), tuple(pad))
    d = L.StemDesc()
    d.n, d.t, d.h, d.wf = 1, t, h, 8 * stem8_mr(w)
    d.cout, d.kt, d.kh, d.kwf = cout, k[0], k[1], g.kwf
    d.str_t, d.str_h, d.pad_t, d.pad_h, d.pad_wf = stride[0], stride[1], pad[0], pad[1], g.pad_wf
    d.out_t, d.out_h, d.out_w = g.out_dims(t, h, w)
    return bool(L.load().sfb_stem8_supported(C.byref(d)))


def stem8_input_fold(x: torch.Tensor, out: Planes) -> None:
    lib = L.load()
    n, c, t, h, w = x.shape
    assert (out.n, out.t, out.h, out.w, out.c) == stem8_plane_dims(n, t, h, w) and out.pitch == 8
    assert x.is_contiguous() and x.dtype == F32
    L.check(lib.sfb_stem8_input_fold(x.data_ptr(), n, c, t, h, w, out.hi_ptr(), out.lo_ptr(), _stream()),
            "sfb_stem8_input_fold")
    _count()


STEM8_ZG = 7 * 12 + 8   # granules per T tap of the zero-flanked filter copy


def stem8_filter_fold(w: torch.Tensor, hi: torch.Tensor, lo: Optional[torch.Tensor]) -> None:
    lib = L.load()
    cout, cin, kt = w.shape[:3]
    assert cout == 8 and hi.numel() == kt * STEM8_ZG * 64 and w.is_contiguous()
    L.check(lib.sfb_stem8_filter_fold(w.data_ptr(), cin, kt, hi.data_ptr(), _ptr(lo), _stream()), "sfb_stem8_filter_fold")
    _count()


def stem8_m_tiles(x: Planes, g: StemGeom) -> int:
    return int(L.load().sfb_stem8_m_tiles(C.byref(_stem8_desc(x, g, 1))))


def stem8_fprop(x: Planes, f_hi: torch.Tensor, f_lo: Optional[torch.Tensor], g: StemGeom, out: torch.Tensor,
                stats: Optional[torch.Tensor], nsplit: int = 3) -> None:
    lib = L.load()
    d = _stem8_desc(x, g, nsplit)
    d.f_hi, d.f_lo = f_hi.data_ptr(), _ptr(f_lo)
    d.out, d.stats = out.data_ptr(), _ptr(stats)
    L.check(lib.sfb_stem8_fprop(C.byref(d), _stream()), "sfb_stem8_fprop")
    _count()


def stem8_wgrad(x: Planes, dy: Planes, g: StemGeom, dwm: torch.Tensor, nsplit: int = 3) -> None:
    lib = L.load()
    assert dy.pitch == dy.c == g.cout == 8
    d = _stem8_desc(x, g, nsplit)
    d.dy_hi, d.dy_lo = dy.hi_ptr(), dy.lo_ptr()
    d.dwm = dwm.data_ptr()
    L.check(lib.sfb_stem8_wgrad(C.byref(d), _stream()), "sfb_stem8_wgrad")
    _count()


# ------------------------------------------------------------------------------------------------ generic max pool
def _pool3d_desc(x: Planes, out_dims, k, s, p):
    d = L.Pool3dDesc()
    d.n, d.t, d.h, d.w, d.c = x.n, x.t, x.h, x.w, x.c
    d.ot, d.oh, d.ow = out_dims
    d.kt, d.kh, d.kw = k
    d.st, d.sh, d.sw = s
    d.pt, d.ph, d.pw = p
    return d


def maxpool3d_fwd(x: Planes, out: Planes, argmax: torch.Tensor, k, s, p) -> None:
    lib = L.load()
    d = _pool3d_desc(x, (out.t, out.h, out.w), k, s, p)
    d.in_hi, d.in_lo, d.in_pitch = x.hi_ptr(), x.lo_ptr(), x.pitch
    d.out_hi, d.out_lo, d.out_pitch = out.hi_ptr(), out.lo_ptr(), out.pitch
    d.argmax = argmax.data_ptr()
    L.check(lib.sfb_maxpool3d_fwd(C.byref(d), _stream()), "sfb_maxpool3d_fwd")
    _count()


def maxpool3d_bwd(dout: F32View, argmax: torch.Tensor, x: Planes, out_dims, din: F32View, k, s, p,
                  accumulate: bool = False) -> None:
    lib = L.load()
    d = _pool3d_desc(x, out_dims, k, s, p)
    d.argmax = argmax.data_ptr()
    d.dout, d.dout_pitch = dout.ptr(), dout.pitch
    d.din, d.din_pitch, d.din_accumulate = din.ptr(), din.pitch, 1 if accumulate else 0
    L.check(lib.sfb_maxpool3d_bwd(C.byref(d), _stream()), "sfb_maxpool3d_bwd")
    _count()


# ------------------------------------------------------------------------------------------------ X3D kernels
@dataclass
class DwGeom:
    """Channelwise Conv3d geometry: input dims, filter, stride, padding -> output dims."""

    n: int
    t: int
    h: int
    w: int
    k: Tuple[int, int, int]
    stride: Tuple[int, int, int]
    pad: Tuple[int, int, int]

    @property
    def out(self) -> Tuple[int, int, int]:
        return tuple(conv_out_size(i, k, s, p) for i, k, s, p in zip((self.t, self.h, self.w), self.k, self.stride,
                                                                     self.pad))


def _dw_desc(g: DwGeom, c: int, c_valid: int, weight: torch.Tensor, x_planes: Optional[Planes] = None,
             x_f32: Optional[F32View] = None, in_affine=None) -> "L.DwConvDesc":
    """``in_affine`` = (scale, shift, relu): the producer's BatchNorm (+ReLU) applied on the fly to an fp32 input."""
    d = L.DwConvDesc()
    if in_affine is not None:
        assert x_f32 is not None
        d.in_scale, d.in_shift, d.in_relu = in_affine[0].data_ptr(), in_affine[1].data_ptr(), 1 if in_affine[2] else 0
    if x_planes is not None:
        assert x_planes.c == c and (x_planes.n, x_planes.t, x_planes.h, x_planes.w) == (g.n, g.t, g.h, g.w)
        d.x_hi, d.x_lo, d.x_pitch = x_planes.hi_ptr(), x_planes.lo_ptr(), x_planes.pitch
    else:
        assert x_f32 is not None and x_f32.c == c and x_f32.rows == g.n * g.t * g.h * g.w
        d.x_f32, d.x_pitch = x_f32.ptr(), x_f32.pitch
    assert weight.is_contiguous() and weight.dtype == F32 and weight.shape[0] == c_valid and weight.shape[1] == 1
    assert tuple(weight.shape[2:]) == tuple(g.k)
    d.w = weight.data_ptr()
    d.n, d.t, d.h, d.w_, d.c, d.c_valid = g.n, g.t, g.h, g.w, c, c_valid
    d.ot, d.oh, d.ow = g.out
    d.kt, d.kh, d.kw = g.k
    d.st, d.sh, d.sw = g.stride
    d.pt, d.ph, d.pw = g.pad
    return d


def dwconv_tiles(g: DwGeom, c: int, f32_input: bool) -> Tuple[int, int]:
    """(m_tiles, tiles_per_sample) of the forward kernel's BatchNorm partials (depends on which kernel the library
    picks for this geometry / input format)."""
    lib = L.load()
    d = L.DwConvDesc()
    d.n, d.t, d.h, d.w_, d.c = g.n, g.t, g.h, g.w, c
    d.ot, d.oh, d.ow = g.out
    d.kt, d.kh, d.kw = g.k
    d.st, d.sh, d.sw = g.stride
    d.pt, d.ph, d.pw = g.pad
    d.x_f32 = 1 if f32_input else None  # only its null-ness matters here
    return lib.sfb_dwconv_m_tiles(C.byref(d)), lib.sfb_dwconv_tiles_per_sample(C.byref(d))


def dwconv_fwd(g: DwGeom, c: int, c_valid: int, weight: torch.Tensor, y: F32View, stats: Optional[torch.Tensor],
               x_planes: Optional[Planes] = None, x_f32: Optional[F32View] = None, in_affine=None) -> None:
    lib = L.load()
    d = _dw_desc(g, c, c_valid, weight, x_planes, x_f32, in_affine)
    assert y.c == c
    d.y, d.y_pitch, d.stats = y.ptr(), y.pitch, _ptr(stats)
    L.check(lib.sfb_dwconv_fwd(C.byref(d), _stream()), "sfb_dwconv_fwd")
    _count()


def dwconv_wgrad_blocks(g: DwGeom) -> int:
    d = L.DwConvDesc()
    d.n = g.n
    d.ot, d.oh, d.ow = g.out
    return L.load().sfb_dwconv_wgrad_blocks(C.byref(d))


def dwconv_bwd(g: DwGeom, c: int, c_valid: int, weight: torch.Tensor, dy: F32View, dw: Optional[torch.Tensor],
               wpartials: Optional[torch.Tensor], x_planes: Optional[Planes] = None,
               x_f32: Optional[F32View] = None, dx: Optional[F32View] = None, dx_planes: Optional[Planes] = None,
               dx_accumulate: bool = False, in_affine=None) -> None:
    lib = L.load()
    d = _dw_desc(g, c, c_valid, weight, x_planes, x_f32, in_affine)
    d.dy, d.dy_pitch = dy.ptr(), dy.pitch
    launches = 0
    if dx is not None:
        assert dx.c == c
        d.dx, d.dx_pitch, d.dx_accumulate = dx.ptr(), dx.pitch, 1 if dx_accumulate else 0
        launches += 1
    elif dx_planes is not None:
        assert dx_planes.c == c
        d.dx_hi, d.dx_lo, d.dx_pitch = dx_planes.hi_ptr(), dx_planes.lo_ptr(), dx_planes.pitch
        launches += 1
    if dw is not None:
        assert dw.is_contiguous() and dw.numel() == weight.numel()
        d.wpartials = _ptr(wpartials)  # (only the generic planes-input kernels need the scratch)
        launches += 2
    L.check(lib.sfb_dwconv_bwd(C.byref(d), _ptr(dw), _stream()), "sfb_dwconv_bwd")
    _count(launches)


ACT_NONE, ACT_RELU, ACT_SWISH = 0, 1, 2


def _bnact_desc(y: F32View, scale, shift, mean, invstd, gate, act: int, rows_per_sample: int) -> "L.BnActDesc":
    d = L.BnActDesc()
    d.y, d.y_pitch = y.ptr(), y.pitch
    d.scale, d.shift, d.mean, d.invstd = scale.data_ptr(), shift.data_ptr(), _ptr(mean), _ptr(invstd)
    d.gate, d.act = _ptr(gate), act
    d.rows, d.rows_per_sample, d.c = y.rows, rows_per_sample, y.c
    return d


def bnact_fwd(y: F32View, scale, shift, gate, act: int, rows_per_sample: int, out: Planes) -> None:
    lib = L.load()
    d = _bnact_desc(y, scale, shift, None, None, gate, act, rows_per_sample)
    assert out.c == y.c and out.rows == y.rows
    d.out_hi, d.out_lo, d.out_pitch = out.hi_ptr(), out.lo_ptr(), out.pitch
    L.check(lib.sfb_bnact_fwd(C.byref(d), _stream()), "sfb_bnact_fwd")
    _count()


def bnact_tiles_per_sample(rows: int, rows_per_sample: int) -> int:
    return L.load().sfb_bnact_tiles_per_sample(rows, rows_per_sample)


def bnact_bwd_reduce(y: F32View, scale, shift, mean, invstd, gate, act: int, rows_per_sample: int, dout: F32View,
                     partials: torch.Tensor) -> None:
    lib = L.load()
    d = _bnact_desc(y, scale, shift, mean, invstd, gate, act, rows_per_sample)
    assert dout.rows == y.rows and dout.c >= y.c
    d.dout, d.dout_pitch, d.partials = dout.ptr(), dout.pitch, partials.data_ptr()
    L.check(lib.sfb_bnact_bwd_reduce(C.byref(d), _stream()), "sfb_bnact_bwd_reduce")
    _count()


def bnact_bwd_apply(y: F32View, scale, shift, mean, invstd, gate, act: int, rows_per_sample: int, dout: F32View,
                    davg, coef, dy: F32View) -> None:
    lib = L.load()
    d = _bnact_desc(y, scale, shift, mean, invstd, gate, act, rows_per_sample)
    d.dout, d.dout_pitch = dout.ptr(), dout.pitch
    d.davg, d.coef = _ptr(davg), coef.data_ptr()
    assert dy.c == y.c and dy.rows == y.rows
    d.dy, d.dy_pitch = dy.ptr(), dy.pitch
    L.check(lib.sfb_bnact_bwd_apply(C.byref(d), _stream()), "sfb_bnact_bwd_apply")
    _count()


def se_fwd(d: "L.SeDesc") -> None:
    L.check(L.load().sfb_se_fwd(C.byref(d), _stream()), "sfb_se_fwd")
    _count()


def se_bwd(d: "L.SeDesc") -> None:
    L.check(L.load().sfb_se_bwd(C.byref(d), _stream()), "sfb_se_bwd")
    _count(2)


def relu_fwd(x: torch.Tensor) -> None:
    assert x.is_contiguous() and x.dtype == F32
    L.check(L.load().sfb_relu_fwd(x.data_ptr(), x.numel(), _stream()), "sfb_relu_fwd")
    _count()


def relu_bwd(dx: torch.Tensor, y: torch.Tensor) -> None:
    assert dx.is_contiguous() and y.is_contiguous() and dx.numel() == y.numel()
    L.check(L.load().sfb_relu_bwd(dx.data_ptr(), y.data_ptr(), dx.numel(), _stream()), "sfb_relu_bwd")
    _count()


def stem_wgrad_direct(x: torch.Tensor, dy: Planes, k, stride, pad, dw: torch.Tensor) -> None:
    """dw[8,3,kt,kh,kw] = weight gradient of the 3 -> 8 channel stem from the fp32 NCTHW clip and the dY planes."""
    lib = L.load()
    n, cin, t, h, w = x.shape
    assert x.dtype == F32 and x.is_contiguous() and dw.is_contiguous() and dy.pitch == dy.c == dw.shape[0]
    L.check(lib.sfb_stem_wgrad_direct(x.data_ptr(), n, cin, t, h, w, dy.hi_ptr(), dy.lo_ptr(), dy.c, k[0], k[1], k[2],
                                      stride[0], stride[1], stride[2], pad[0], pad[1], pad[2], dw.data_ptr(),
                                      _stream()), "sfb_stem_wgrad_direct")
    _count(2)


# ------------------------------------------------------------------------------------------------ batched filter packing
class PackPlan:
    """All filter packs of one phase (forward / backward) of a model step as ONE kernel launch.

    During the first pass of a phase the engine packs layer by layer (``filter_pack``) and ``record``s each job; from
    the second pass on ``launch`` replays the whole list with ``sfb_filter_pack_multi``.  A job is (weight, FilterMat,
    tapmap, transpose); the packed buffers must be persistent (not shared scratch)."""

    ITEMS_PER_BLOCK = 256 * 16  # grid-stride work per block of 256 threads

    def __init__(self):
        self.jobs = []          # (weight tensor, FilterMat, tapmap tuple | None, transpose)
        self._table = None      # device uint8 tensor holding the sfb_pack_job array
        self._sig = None
        self.total_blocks = 0

    def record(self, w: torch.Tensor, out: "FilterMat", tapmap, transpose: bool) -> bool:
        ntaps = out.ntaps
        if ntaps > 32:
            return False  # (stems) stays an individual launch
        self.jobs.append((w, out, None if tapmap is None else tuple(int(t) for t in tapmap), bool(transpose)))
        self._table = None
        return True

    def signature(self):
        return tuple((w.data_ptr(), o.hi.data_ptr(), None if o.lo is None else o.lo.data_ptr()) for w, o, _, _ in self.jobs)

    @staticmethod
    def job_blocks(rows: int, ntaps: int, cols_pad: int) -> int:
        items = rows * ntaps * cols_pad
        return max(1, min(64, (items + PackPlan.ITEMS_PER_BLOCK - 1) // PackPlan.ITEMS_PER_BLOCK))

    def build_table(self):
        """ctypes array of sfb_pack_job (host side); returns (array, total_blocks)."""
        arr = (L.PackJob * len(self.jobs))()
        first = 0
        for k, (w, out, tapmap, transpose) in enumerate(self.jobs):
            cout, cin = w.shape[0], w.shape[1]
            taps_total = w[0, 0].numel() if w.dim() > 2 else 1
            j = arr[k]
            j.w, j.hi, j.lo = w.data_ptr(), out.hi.data_ptr(), _ptr(out.lo)
            j.cout, j.cin, j.taps_total, j.ntaps = cout, cin, taps_total, out.ntaps
            j.transpose, j.cols_pad = 1 if transpose else 0, out.cols_pad
            tm = tapmap if tapmap is not None else tuple(range(out.ntaps))
            assert len(tm) == out.ntaps and all(0 <= t < taps_total for t in tm)
            for i, t in enumerate(tm):
                j.tapmap[i] = t
            rows = cin if transpose else cout
            j.first_block = first
            j.n_blocks = self.job_blocks(rows, out.ntaps, out.cols_pad)
            first += j.n_blocks
        return arr, first

    def finalize(self, device) -> None:
        arr, total = self.build_table()
        raw = bytes(arr)
        self._table = torch.frombuffer(bytearray(raw), dtype=torch.uint8).to(device)
        self.total_blocks = total
        self._sig = self.signature()

    @property
    def ready(self) -> bool:
        return self._table is not None and len(self.jobs) > 0

    def launch(self) -> None:
        assert self.ready
        L.check(L.load().sfb_filter_pack_multi(self._table.data_ptr(), len(self.jobs), self.total_blocks, _stream()),
                "sfb_filter_pack_multi")
        _count()
