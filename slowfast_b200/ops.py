"""Torch-tensor front end of the C ABI (``include/slowfast_b200.h``).

PyTorch is used for device memory, streams and dtype bookkeeping only; every function here enqueues one or more
of the library's own kernels on the current CUDA stream.  The model programs (``nets/``) launch the library only through
these functions, which fill the descriptors, check the return code and count the launches; the optimizer and the uint8
input pipeline keep their own single calls.  There is no CPU path: without the native library or a
CUDA device the calls raise ``NativeLibraryError``.
"""
from __future__ import annotations

import ctypes as C
import math
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
    """128-row output tiles of a convolution (the tile rows of an unsplit launch).  The BatchNorm partials of a launch
    have ``conv_stats_tiles`` columns."""
    m = n * geom.out[0] * geom.out[1] * geom.out[2]
    return (m + 127) // 128


def _conv_desc(x: Planes, f: FilterMat, geom: ConvGeom, out: torch.Tensor, out_strides: Tuple[int, int, int, int],
               out_offset: int, accumulate, stats: Optional[torch.Tensor], nsplit: int):
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
    return d


def conv_stats_tiles(x: Planes, f: FilterMat, geom: ConvGeom, out: torch.Tensor,
                     out_strides: Tuple[int, int, int, int], out_offset: int = 0, nsplit: int = 3) -> int:
    """Columns of the BatchNorm partials ``[2][f.rows][columns]`` that ``conv_igemm`` writes for these arguments
    with ``stats`` (a split-K launch takes them from its output afterwards, in its own row blocks)."""
    d = _conv_desc(x, f, geom, out, out_strides, out_offset, 0, None, nsplit)
    return int(L.load().sfb_conv_m_tiles(C.byref(d)))


def conv_ksplit(x: Planes, f: FilterMat, geom: ConvGeom, out: torch.Tensor, out_strides: Tuple[int, int, int, int],
                out_offset: int = 0, accumulate=0, stats: Optional[torch.Tensor] = None, nsplit: int = 3) -> int:
    """CTAs per output tile (split-K slices) that ``conv_igemm`` would use for these arguments; 1 = no split."""
    d = _conv_desc(x, f, geom, out, out_strides, out_offset, accumulate, stats, nsplit)
    return int(L.load().sfb_conv_ksplit(C.byref(d)))


def conv_igemm(x: Planes, f: FilterMat, geom: ConvGeom, out: torch.Tensor, out_strides: Tuple[int, int, int, int],
               out_offset: int = 0, accumulate: bool = False, stats: Optional[torch.Tensor] = None,
               nsplit: int = 3) -> None:
    """out view[n, z, p, q, :f.rows] (+)= conv(x, f).  ``out_strides`` are element strides for (n, t, h, w);
    ``out_offset`` an element offset into ``out`` (channel slice / strided scatter).  ``stats``: BatchNorm partials
    ``[2][f.rows][conv_stats_tiles(...)]``."""
    lib = L.load()
    d = _conv_desc(x, f, geom, out, out_strides, out_offset, accumulate, stats, nsplit)
    L.check(lib.sfb_conv_igemm(C.byref(d), _stream()), "sfb_conv_igemm")
    _count()


def _wgrad_desc(x: Planes, dy: Planes, geom: ConvGeom, dwm: Optional[torch.Tensor], nsplit: int):
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
    d.dw = _ptr(dwm)
    d.nsplit = nsplit
    return d


def conv_wgrad_plan(x: Planes, dy: Planes, geom: ConvGeom, nsplit: int = 3, num_sms: Optional[int] = None):
    """The tiling ``conv_wgrad`` uses for these operands on a device with ``num_sms`` multiprocessors (default: the
    current device's).  Needs no device when ``num_sms`` is given."""
    if num_sms is None:
        num_sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    plan = L.WgradPlan()
    L.check(L.load().sfb_conv_wgrad_plan(C.byref(_wgrad_desc(x, dy, geom, None, nsplit)), num_sms, C.byref(plan)),
            "sfb_conv_wgrad_plan")
    return plan


def conv_wgrad(x: Planes, dy: Planes, geom: ConvGeom, dwm: torch.Tensor, nsplit: int = 3) -> None:
    """dwm[cout, taps*x.c] += dY^T * im2col(x).  dy must be dense rows [M, cout] (its pitch may exceed cout)."""
    lib = L.load()
    d = _wgrad_desc(x, dy, geom, dwm, nsplit)
    L.check(lib.sfb_conv_wgrad(C.byref(d), _stream()), "sfb_conv_wgrad")
    _count()


# ------------------------------------------------------------------------------------------------ batch norm
def bn_finalize(partials: Optional[torch.Tensor], m_tiles: int, c: int, count: int, gamma, beta, running_mean,
                running_var, momentum: float, eps: float, training: bool, scale, shift, save_mean, save_invstd,
                affine_c: int = 0):
    """``affine_c``: period of gamma / beta (sub-batch BN: ``c`` = S*C split channels share one [C] affine)."""
    lib = L.load()
    L.check(lib.sfb_bn_finalize(_ptr(partials), m_tiles, c, count, _ptr(gamma), _ptr(beta), _ptr(running_mean),
                                _ptr(running_var), momentum, eps, 1 if training else 0, scale.data_ptr(),
                                shift.data_ptr(), _ptr(save_mean), _ptr(save_invstd), affine_c, _stream()),
            "sfb_bn_finalize")
    _count()


def bn_split_stats_tiles(rows: int, rows_per_clip: int, splits: int, c: int) -> int:
    """Partial columns per split channel that ``bn_split_stats`` writes for a ``c``-channel activation."""
    return L.load().sfb_bn_split_stats_tiles(rows, rows_per_clip, splits, c)


def bn_split_stats(y: F32View, splits: int, rows_per_clip: int, partials: torch.Tensor) -> None:
    """Sub-batch BN training statistics of y: partials [2][splits*c][bn_split_stats_tiles(...)] for ``bn_finalize``
    over ``splits*c`` channels (clip k is split k % splits)."""
    lib = L.load()
    tiles = bn_split_stats_tiles(y.rows, rows_per_clip, splits, y.c)
    assert partials.dtype == F32 and partials.numel() >= 2 * splits * y.c * tiles
    L.check(lib.sfb_bn_split_stats(y.ptr(), y.pitch, y.rows, y.c, splits, rows_per_clip, partials.data_ptr(),
                                   _stream()), "sfb_bn_split_stats")
    _count()


def bn_apply(y: F32View, scale, shift, out: Planes, relu: bool, y2: Optional[F32View] = None, scale2=None,
             shift2=None, res: Optional[Planes] = None, splits: int = 1, rows_per_clip: int = 0) -> None:
    """``splits`` > 1: scale / shift (scale2 / shift2) are [splits][c] tables, row r uses row
    (r // rows_per_clip) % splits."""
    lib = L.load()
    d = L.BnApplyDesc()
    d.splits, d.rows_per_clip = splits, rows_per_clip
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


def bn_bwd_blocks(rows: int, c: int, splits: int = 1, rows_per_clip: int = 0) -> int:
    return L.load().sfb_bn_bwd_blocks(rows, c, splits, rows_per_clip)


def bn_bwd_scratch(rows: int, c: int, device, splits: int = 1, rows_per_clip: int = 0):
    nb = bn_bwd_blocks(rows, c, splits, rows_per_clip)
    return (torch.empty((nb, 2, c), dtype=F32, device=device), torch.empty((3, splits * c), dtype=F32, device=device))


def bn_bwd(dout: F32View, mask: Optional[Planes], y: F32View, mean, invstd, gamma, dgamma, dbeta, dy: Planes,
           partials, coef, training: bool = True, accumulate_param_grads: bool = False,
           dres: Optional[F32View] = None, dres_accumulate: bool = False, c_valid: int = 0,
           mask_affine=None, splits: int = 1, rows_per_clip: int = 0) -> None:
    """``mask``: post-ReLU planes (ReLU mask = planes > 0) or None; ``mask_affine`` = (scale, shift): recompute the
    mask as y*scale + shift > 0 instead (used when the activation was never materialised).  ``splits`` > 1: mean /
    invstd (and mask_affine) are [splits][c] tables of sub-batch BN, clip k of the batch being split k % splits."""
    lib = L.load()
    d = L.BnBwdDesc()
    d.c_valid = c_valid
    d.splits, d.rows_per_clip = splits, rows_per_clip
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


def bn_relu_maxpool_fwd(y: torch.Tensor, scale, shift, out: Planes, argmax: torch.Tensor, k, s, p,
                        splits: int = 1) -> None:
    """``splits`` > 1: scale / shift are [splits][c] tables, clip n uses row n % splits."""
    lib = L.load()
    n, t, h, w, c = y.shape
    d = _pool_desc(n, t, h, w, c, out.h, out.w, k, s, p)
    d.splits = splits
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


def small_linear_fwd(x, w, b, y, relu: bool = False) -> None:
    """y = x w^T + b; ``relu``: y = relu(x w^T + b) in the same pass."""
    lib = L.load()
    m, j = x.shape
    k = w.shape[0]
    name = "sfb_small_linear_relu_fwd" if relu else "sfb_small_linear_fwd"
    L.check(getattr(lib, name)(x.data_ptr(), w.data_ptr(), _ptr(b), y.data_ptr(), m, k, j, _stream()), name)
    _count()


def small_linear_bwd(dy, x, w, dw, db, dx, accumulate: bool = False, relu_mask: bool = False) -> None:
    """``relu_mask``: x is the output of a ReLU, and dx is the gradient at that ReLU's input (zero where x <= 0)."""
    lib = L.load()
    m, j = x.shape
    k = w.shape[0]
    name = "sfb_small_linear_relu_bwd" if relu_mask else "sfb_small_linear_bwd"
    L.check(getattr(lib, name)(dy.data_ptr(), x.data_ptr(), w.data_ptr(), _ptr(dw), _ptr(db), _ptr(dx), m, k, j,
                               1 if accumulate else 0, _stream()), name)
    _count((1 if dw is not None else 0) + (1 if dx is not None else 0))


MOMENTUM_CHUNK = 8192  # elements per thread block of sfb_momentum_update


def momentum_table(pairs: Sequence[Tuple[torch.Tensor, torch.Tensor]]) -> torch.Tensor:
    """Device chunk table of sfb_momentum_update for (query, key) parameter pairs; it holds their current pointers."""
    lib = L.load()
    assert lib.sfb_momentum_chunk_size() == C.sizeof(L.MomentumChunk)
    chunks = []
    for q, k in pairs:
        assert q.shape == k.shape and q.dtype == k.dtype == F32 and q.is_contiguous() and k.is_contiguous()
        assert q.device == k.device and k.is_cuda
        n = k.numel()
        for c0 in range(0, n, MOMENTUM_CHUNK):
            chunks.append((k.data_ptr() + 4 * c0, q.data_ptr() + 4 * c0, min(MOMENTUM_CHUNK, n - c0)))
    arr = (L.MomentumChunk * len(chunks))()
    for i, (kp, qp, cnt) in enumerate(chunks):
        arr[i].key, arr[i].query, arr[i].count = kp, qp, cnt
    return torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).to(pairs[0][1].device)


def momentum_update(table: torch.Tensor, m: float) -> None:
    """key = query * (1 - m) + key * m in place over every chunk of ``table`` (``momentum_table``).  The coefficients
    are rounded to fp32 the way ATen rounds a Python scalar: 1 - m in double first."""
    lib = L.load()
    n = table.numel() // C.sizeof(L.MomentumChunk)
    L.check(lib.sfb_momentum_update(table.data_ptr(), n, 1.0 - float(m), float(m), _stream()), "sfb_momentum_update")
    _count()


def row_softmax(x: torch.Tensor) -> None:
    lib = L.load()
    L.check(lib.sfb_row_softmax(x.data_ptr(), x.shape[0], x.shape[1], _stream()), "sfb_row_softmax")
    _count()


def row_sigmoid(x: torch.Tensor) -> None:
    lib = L.load()
    L.check(lib.sfb_row_sigmoid(x.data_ptr(), x.shape[0], x.shape[1], _stream()), "sfb_row_sigmoid")
    _count()


HEAD_ACTS = ("softmax", "sigmoid", "none")


def head_act(x: torch.Tensor, act_func: str) -> None:
    """The eval-mode activation of a classification head (MODEL.HEAD_ACT) in place on the [rows, classes] output."""
    if act_func == "softmax":
        row_softmax(x)
    elif act_func == "sigmoid":
        row_sigmoid(x)
    else:
        assert act_func == "none", act_func


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
    """W-shift stem forward (csrc/conv_stem.cu): up to 64 output channels (one accumulator tile of 16, 32, 48 or 64
    columns); the stems of the supported models have 8, 24 or 64."""
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


# ------------------------------------------------------------------------------------------------ row / batched-GEMM pieces
def colsum_blocks(rows: int) -> int:
    """Row slabs of ``colsum``'s partial sums (first extent of its ``partials`` scratch)."""
    return int(L.load().sfb_rowslab_blocks(rows))


def colsum(src: torch.Tensor, rows: int, c: int, out: torch.Tensor, partials: torch.Tensor, pitch: Optional[int] = None,
           accumulate: bool = False) -> None:
    """out[c] (= or +=) column sums of the fp32 matrix src[rows, c] (row pitch ``pitch``): bias gradients.
    ``partials``: fp32 scratch of at least colsum_blocks(rows) * c elements."""
    lib = L.load()
    assert partials.numel() >= colsum_blocks(rows) * c
    L.check(lib.sfb_colsum(src.data_ptr(), pitch or c, rows, c, out.data_ptr(), 1 if accumulate else 0,
                           partials.data_ptr(), _stream()), "sfb_colsum")
    _count(2)


def gemm_batched(a: Planes, a_shape, a_mn: bool, b: Planes, b_shape, b_mn: bool, m: int, n: int, k: int, batch: int,
                 out: torch.Tensor, ldd: int, alpha: float = 1.0, accumulate: bool = False, nsplit: int = 3) -> None:
    """out[b](m, n) (+)= alpha * sum_k A[b](m, k) * B[b](n, k) (csrc/gemm_batched.cu); a_shape / b_shape = (pitch,
    batch stride) in elements of the operand planes as laid out in memory, *_mn: operand stored MN-major."""
    lib = L.load()
    d = L.BgemmDesc()
    d.a_hi, d.a_lo, d.lda, d.batch_stride_a, d.a_mn_major = a.hi_ptr(), a.lo_ptr(), a_shape[0], a_shape[1], int(a_mn)
    d.b_hi, d.b_lo, d.ldb, d.batch_stride_b, d.b_mn_major = b.hi_ptr(), b.lo_ptr(), b_shape[0], b_shape[1], int(b_mn)
    d.m, d.n, d.k, d.batch = m, n, k, batch
    d.out, d.ldd, d.batch_stride_d = out.data_ptr(), ldd, m * ldd
    d.alpha, d.accumulate, d.nsplit = alpha, 1 if accumulate else 0, nsplit
    L.check(lib.sfb_gemm_batched(C.byref(d), _stream()), "sfb_gemm_batched")
    _count()


def bias_split(x: F32View, bias: Optional[torch.Tensor], out: Planes) -> None:
    """planes[rows, out.c] = x[rows, x.c] (+ bias), columns past x.c zero (csrc/nonlocal.cu)."""
    lib = L.load()
    assert x.rows == out.rows and x.c <= out.c
    assert bias is None or (bias.is_contiguous() and bias.numel() == x.c)
    L.check(lib.sfb_bias_split(x.ptr(), x.rows, x.c, x.pitch, _ptr(bias), out.hi_ptr(), out.lo_ptr(), out.pitch, out.c,
                               _stream()), "sfb_bias_split")
    _count()


def bn_conv_bias(bias: torch.Tensor, c: int, momentum: float, training: bool, running_mean, scale, shift,
                 save_mean, splits: int = 1) -> None:
    """Fold a conv bias into the BatchNorm that follows it, after ``bn_finalize`` (csrc/nonlocal.cu).  ``splits`` > 1:
    running_mean is a sub-batch BN's [splits][c] split_bn statistics (training)."""
    lib = L.load()
    L.check(lib.sfb_bn_conv_bias(bias.data_ptr(), c, momentum, 1 if training else 0, _ptr(running_mean), _ptr(scale),
                                 _ptr(shift), _ptr(save_mean), splits, _stream()), "sfb_bn_conv_bias")
    _count()


def planes_to_f32(x: Planes, out: F32View) -> None:
    lib = L.load()
    assert out.rows == x.rows and out.c == x.c
    L.check(lib.sfb_planes_to_f32(x.hi_ptr(), x.lo_ptr(), x.rows, x.c, x.pitch, out.ptr(), out.pitch, _stream()),
            "sfb_planes_to_f32")
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


def _dw_desc(g: DwGeom, c: int, c_valid: int, weight: torch.Tensor, x_f32: F32View, in_affine=None) -> "L.DwConvDesc":
    """``in_affine`` = (scale, shift, relu): the producer's BatchNorm (+ReLU) applied on the fly to the input."""
    d = L.DwConvDesc()
    if in_affine is not None:
        d.in_scale, d.in_shift, d.in_relu = in_affine[0].data_ptr(), in_affine[1].data_ptr(), 1 if in_affine[2] else 0
    assert x_f32.c == c and x_f32.rows == g.n * g.t * g.h * g.w
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


def dwconv_tiles(g: DwGeom, c: int) -> Tuple[int, int]:
    """(m_tiles, tiles_per_sample) of the forward kernel's BatchNorm partials (depends on which kernel the library
    picks for this geometry)."""
    lib = L.load()
    d = L.DwConvDesc()
    d.n, d.t, d.h, d.w_, d.c = g.n, g.t, g.h, g.w, c
    d.ot, d.oh, d.ow = g.out
    d.kt, d.kh, d.kw = g.k
    d.st, d.sh, d.sw = g.stride
    d.pt, d.ph, d.pw = g.pad
    return lib.sfb_dwconv_m_tiles(C.byref(d)), lib.sfb_dwconv_tiles_per_sample(C.byref(d))


def dwconv_fwd(g: DwGeom, c: int, c_valid: int, weight: torch.Tensor, y: F32View, stats: Optional[torch.Tensor],
               x_f32: F32View, in_affine=None) -> None:
    lib = L.load()
    d = _dw_desc(g, c, c_valid, weight, x_f32, in_affine)
    assert y.c == c
    d.y, d.y_pitch, d.stats = y.ptr(), y.pitch, _ptr(stats)
    L.check(lib.sfb_dwconv_fwd(C.byref(d), _stream()), "sfb_dwconv_fwd")
    _count()


def dwconv_bwd(g: DwGeom, c: int, c_valid: int, weight: torch.Tensor, dy: F32View, dw: Optional[torch.Tensor],
               x_f32: F32View, dx: Optional[F32View] = None, dx_planes: Optional[Planes] = None,
               dx_accumulate: bool = False, in_affine=None) -> None:
    lib = L.load()
    d = _dw_desc(g, c, c_valid, weight, x_f32, in_affine)
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
        launches += 2  # memset + kernel
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


# ------------------------------------------------------------------------------------------------ token path (MViT / ViT)
def layernorm_fwd(x: torch.Tensor, x_pitch: int, rows: int, c: int, weight, bias, eps: float, mean, rstd,
                  out: Optional[Planes] = None, out_f32: Optional[torch.Tensor] = None) -> None:
    """LayerNorm of the c channels of every row of x (row pitch ``x_pitch``) -> planes ``out`` and / or the dense fp32
    [rows, c] ``out_f32``; mean / rstd [rows] are kept for the backward."""
    assert out is None or (out.rows == rows and out.c == c and out.pitch == c)
    L.check(L.load().sfb_layernorm_fwd(x.data_ptr(), x_pitch, rows, c, weight.data_ptr(), bias.data_ptr(), eps,
                                       None if out is None else out.hi_ptr(), None if out is None else out.lo_ptr(),
                                       _ptr(out_f32), c, mean.data_ptr(), rstd.data_ptr(), _stream()), "sfb_layernorm_fwd")
    _count()


def layernorm_bwd(dy: torch.Tensor, dy_pitch: int, x: torch.Tensor, x_pitch: int, rows: int, c: int, weight, mean, rstd,
                  dx: torch.Tensor, dx_pitch: int, dweight, dbias, partials: torch.Tensor, dx_accumulate: bool = False,
                  param_accumulate: bool = False) -> None:
    """dx (+)= LayerNorm backward of dy; dweight / dbias (+)= the parameter gradients.  ``partials``: fp32 scratch of at
    least colsum_blocks(rows) * 2 * c elements."""
    assert partials.numel() >= colsum_blocks(rows) * 2 * c
    L.check(L.load().sfb_layernorm_bwd(dy.data_ptr(), dy_pitch, x.data_ptr(), x_pitch, rows, c, weight.data_ptr(),
                                       mean.data_ptr(), rstd.data_ptr(), dx.data_ptr(), dx_pitch, int(dx_accumulate),
                                       dweight.data_ptr(), dbias.data_ptr(), int(param_accumulate), partials.data_ptr(),
                                       _stream()), "sfb_layernorm_bwd")
    _count(2)


def tokens_assemble(y: torch.Tensor, bias, cls, pos_spatial, pos_temporal, pos_class, b: int, lt: int, hw: int, e: int,
                    out: torch.Tensor) -> None:
    """out[b, 1 + lt, e] = [cls ; y + bias] (+ the separable position tables: spatial [hw, e] in every frame, temporal
    [lt / hw, e], class [e]; all three or none)."""
    L.check(L.load().sfb_tokens_assemble(y.data_ptr(), bias.data_ptr(), cls.data_ptr(), _ptr(pos_spatial),
                                         _ptr(pos_temporal), _ptr(pos_class), b, lt, hw, e, out.data_ptr(), _stream()),
            "sfb_tokens_assemble")
    _count()


def tokens_assemble_joint(y: torch.Tensor, bias, cls, pos, b: int, lt: int, e: int, out: torch.Tensor) -> None:
    """out = [cls ;] y + bias (+ pos, the joint [(cls +) lt, e] table): the cls-free layout when ``cls`` is None."""
    L.check(L.load().sfb_tokens_assemble_joint(y.data_ptr(), bias.data_ptr(), _ptr(cls), _ptr(pos), b, lt, e,
                                               out.data_ptr(), _stream()), "sfb_tokens_assemble_joint")
    _count()


def tokens_split_grad(dx: torch.Tensor, b: int, lt: int, e: int, dy: Planes, dy_f32: torch.Tensor) -> None:
    """Gradient of the [b, 1 + lt, e] token sequence -> the patch embedding's output gradient without the cls rows
    (planes + fp32 [b * lt, e])."""
    assert dy.rows == b * lt and dy.c == e and dy.pitch == e
    L.check(L.load().sfb_tokens_split_grad(dx.data_ptr(), b, lt, e, dy.hi_ptr(), dy.lo_ptr(), dy_f32.data_ptr(),
                                           _stream()), "sfb_tokens_split_grad")
    _count()


def segment_slabs(segments: int, length: int) -> int:
    """Row slabs per segment of the deterministic segment sums (token means, position gradients)."""
    return int(L.load().sfb_segment_slabs(segments, length))


def pos_embed_sep_bwd(dx: torch.Tensor, b: int, t: int, hw: int, e: int, dspatial, dtemporal, dclass,
                      partials: torch.Tensor) -> None:
    """Gradients of the separable position tables from the token gradient [b, 1 + t * hw, e].  ``partials``: fp32
    scratch of at least t * segment_slabs(t, hw) * e elements."""
    assert partials.numel() >= t * segment_slabs(t, hw) * e
    L.check(L.load().sfb_pos_embed_sep_bwd(dx.data_ptr(), b, t, hw, e, dspatial.data_ptr(), dtemporal.data_ptr(),
                                           dclass.data_ptr(), partials.data_ptr(), _stream()), "sfb_pos_embed_sep_bwd")
    _count(3)


def pos_embed_joint_bwd(dx: torch.Tensor, b: int, n: int, e: int, dpos) -> None:
    """dpos[n, e] = sum over the batch of the token gradient [b, n, e]."""
    L.check(L.load().sfb_pos_embed_joint_bwd(dx.data_ptr(), b, n, e, dpos.data_ptr(), _stream()),
            "sfb_pos_embed_joint_bwd")
    _count()


def token_mean_fwd(x: torch.Tensor, b: int, n: int, c: int, out: torch.Tensor, partials: torch.Tensor,
                   cls: bool = True) -> None:
    """out[b, c] = mean over the tokens of x [b, n, c], the cls row (``cls``) excluded.  ``partials``: fp32 scratch of at
    least b * segment_slabs(b, n - cls) * c elements."""
    assert partials.numel() >= b * segment_slabs(b, n - int(cls)) * c
    lib = L.load()
    fn, name = (lib.sfb_token_mean_fwd, "sfb_token_mean_fwd") if cls else (lib.sfb_token_mean_all_fwd,
                                                                           "sfb_token_mean_all_fwd")
    L.check(fn(x.data_ptr(), b, n, c, out.data_ptr(), partials.data_ptr(), _stream()), name)
    _count(2)


def token_mean_bwd(dout: torch.Tensor, b: int, n: int, c: int, dx: torch.Tensor, cls: bool = True) -> None:
    """dx[b, n, c] = dout / (n - cls) on every averaged token (zero on the cls row)."""
    lib = L.load()
    fn, name = (lib.sfb_token_mean_bwd, "sfb_token_mean_bwd") if cls else (lib.sfb_token_mean_all_bwd,
                                                                           "sfb_token_mean_all_bwd")
    L.check(fn(dout.data_ptr(), b, n, c, dx.data_ptr(), _stream()), name)
    _count()


def patchify(x: torch.Tensor, k: Sequence[int], out: Planes) -> None:
    """Non-overlapping patches (stride == kernel k) of the NCTHW fp32 clip -> planes [n * patches, cin * kt * kh * kw]."""
    n, cin, t, h, w = x.shape
    assert x.dtype == F32 and x.is_contiguous() and out.pitch == out.c == cin * k[0] * k[1] * k[2]
    assert out.rows == n * (t // k[0]) * (h // k[1]) * (w // k[2])
    L.check(L.load().sfb_patchify(x.data_ptr(), n, cin, t, h, w, *k, out.hi_ptr(), out.lo_ptr(), _stream()),
            "sfb_patchify")
    _count()


def patchify_gather(x: torch.Tensor, k: Sequence[int], ids_keep: Optional[torch.Tensor], keep: int, out: Planes) -> None:
    """``patchify`` of the ``keep`` patches per clip listed in ids_keep [n, keep] (int32); a null ``ids_keep`` packs every
    patch."""
    n, cin, t, h, w = x.shape
    assert x.dtype == F32 and x.is_contiguous() and out.pitch == out.c == cin * k[0] * k[1] * k[2]
    L.check(L.load().sfb_patchify_gather(x.data_ptr(), n, cin, t, h, w, *k, _ptr(ids_keep), keep, out.hi_ptr(),
                                         out.lo_ptr(), _stream()), "sfb_patchify_gather")
    _count()


def _dwpool_desc(src: torch.Tensor, src_c0: int, bias, weight, b, heads, hd, thw, othw, kernel, stride, cls):
    """Pooling of one third (channels src_c0 ..) of the fused qkv rows src [b, cls + thw, pitch]; ``weight`` None: no
    pooling, the third is copied (+ bias) into the head-major layout."""
    d = L.DwPoolDesc()
    d.src, d.src_pitch, d.src_c0 = src.data_ptr(), src.shape[-1], src_c0
    d.bias = _ptr(bias)
    d.b, d.heads, d.hd = b, heads, hd
    d.t, d.h, d.w_ = thw
    d.ot, d.oh, d.ow = othw
    d.has_pool = 1 if weight is not None else 0
    d.no_cls = 0 if cls else 1
    if weight is not None:
        d.w = weight.data_ptr()
        d.kt, d.kh, d.kw = kernel
        d.st, d.sh, d.sw = stride
    else:
        d.kt = d.kh = d.kw = d.st = d.sh = d.sw = 1
    return d


def dwpool_fwd(src: torch.Tensor, src_c0: int, bias, weight, b: int, heads: int, hd: int, thw, othw, kernel, stride,
               out: torch.Tensor, cls: bool = True) -> None:
    """out[b, heads, cls + othw, hd] = depthwise Conv3d (``weight`` [hd, 1, *kernel], padding kernel // 2, shared by the
    heads) of one third of the fused qkv rows (+ its bias); the cls row passes through."""
    d = _dwpool_desc(src, src_c0, bias, weight, b, heads, hd, thw, othw, kernel, stride, cls)
    d.out = out.data_ptr()
    L.check(L.load().sfb_dwpool_fwd(C.byref(d), _stream()), "sfb_dwpool_fwd")
    _count()


def dwpool_wgrad_blocks(b: int, heads: int, othw) -> int:
    """Blocks of ``dwpool_bwd``'s weight-gradient partial sums (its ``wpartials`` holds blocks * hd * taps floats)."""
    d = L.DwPoolDesc()
    d.b, d.heads = b, heads
    d.ot, d.oh, d.ow = othw
    return int(L.load().sfb_dwpool_wgrad_blocks(C.byref(d)))


def dwpool_bwd(src: torch.Tensor, src_c0: int, bias, weight, b: int, heads: int, hd: int, thw, othw, kernel, stride,
               dout: torch.Tensor, dsrc: torch.Tensor, dw: Optional[torch.Tensor] = None,
               wpartials: Optional[torch.Tensor] = None, cls: bool = True) -> None:
    """dsrc (same layout as src, only this third is touched) += the data gradient of ``dwpool_fwd``; dw = its weight
    gradient (pooled thirds, with the ``wpartials`` scratch)."""
    d = _dwpool_desc(src, src_c0, bias, weight, b, heads, hd, thw, othw, kernel, stride, cls)
    d.dout, d.dsrc = dout.data_ptr(), dsrc.data_ptr()
    assert (dw is None) == (weight is None)
    if weight is not None:
        assert wpartials.numel() >= dwpool_wgrad_blocks(b, heads, othw) * hd * math.prod(kernel)
        d.wpartials = wpartials.data_ptr()
    L.check(L.load().sfb_dwpool_bwd(C.byref(d), _ptr(dw), 0, _stream()), "sfb_dwpool_bwd")
    _count(3 if weight is not None else 1)


def softmax_relpos_fwd(s: torch.Tensor, p: Planes, bh: int, nq: int, nk: int, q_thw=(1, 1, 1), k_thw=(1, 1, 1),
                       rq: Optional[torch.Tensor] = None, cls: bool = True, spatial_only: bool = False) -> None:
    """P = softmax over the nk keys of every row of S [bh * nq, pitch] -> planes (pad columns zero), with the decomposed
    relative-position bias gathered from RQ [bh * (nq - cls), pitch] for the query / key grids q_thw / k_thw (Rt
    columns absent when ``spatial_only``; the cls row and column get no bias).  Without ``rq``: a plain row softmax."""
    d = L.SoftmaxDesc()
    d.s, d.s_pitch = s.data_ptr(), s.shape[-1]
    if rq is not None:
        d.rq, d.rq_pitch = rq.data_ptr(), rq.shape[-1]
    d.p_hi, d.p_lo, d.p_pitch = p.hi_ptr(), p.lo_ptr(), p.pitch
    d.bh, d.nq, d.nk = bh, nq, nk
    d.qt, d.qh, d.qw = q_thw
    d.kt, d.kh, d.kw = k_thw
    d.no_cls, d.spatial_only = 0 if cls else 1, int(spatial_only)
    L.check(L.load().sfb_softmax_relpos_fwd(C.byref(d), _stream()), "sfb_softmax_relpos_fwd")
    _count()


def softmax_relpos_bwd(p: Planes, dp: torch.Tensor, ds: Planes, bh: int, nq: int, nk: int, q_thw=(1, 1, 1),
                       k_thw=(1, 1, 1), drq: Optional[torch.Tensor] = None, cls: bool = True,
                       spatial_only: bool = False) -> None:
    """dS = P * (dP - sum_k P dP) -> planes (pad columns zero); ``drq`` receives dS scattered onto the table columns."""
    d = L.SoftmaxDesc()
    d.p_hi, d.p_lo, d.p_pitch = p.hi_ptr(), p.lo_ptr(), p.pitch
    d.dp, d.dp_pitch = dp.data_ptr(), dp.shape[-1]
    d.ds_hi, d.ds_lo, d.ds_pitch = ds.hi_ptr(), ds.lo_ptr(), ds.pitch
    if drq is not None:
        d.drq, d.rq_pitch = drq.data_ptr(), drq.shape[-1]
    d.bh, d.nq, d.nk = bh, nq, nk
    d.qt, d.qh, d.qw = q_thw
    d.kt, d.kh, d.kw = k_thw
    d.no_cls, d.spatial_only = 0 if cls else 1, int(spatial_only)
    L.check(L.load().sfb_softmax_relpos_bwd(C.byref(d), _stream()), "sfb_softmax_relpos_bwd")
    _count()


def attn_merge(o: torch.Tensor, q: Planes, b: int, heads: int, nq: int, hd: int, residual: bool, out: Planes,
               cls: bool = True) -> None:
    """Head-major attention output O [b * heads, nq, hd] (+ the pooled q: residual pooling) -> token rows [b * nq,
    heads * hd] (planes)."""
    lib = L.load()
    fn, name = (lib.sfb_attn_merge, "sfb_attn_merge") if cls else (lib.sfb_attn_merge_nocls, "sfb_attn_merge_nocls")
    L.check(fn(o.data_ptr(), q.hi_ptr(), q.lo_ptr(), b, heads, nq, hd, int(residual), out.hi_ptr(), out.lo_ptr(),
               _stream()), name)
    _count()


def attn_split_grad(dmerged: torch.Tensor, b: int, heads: int, nq: int, hd: int, residual: bool, do: Planes,
                    dq: torch.Tensor, cls: bool = True) -> None:
    """The backward of ``attn_merge``: dO planes and (residual pooling) dq [b * heads, nq, hd]."""
    lib = L.load()
    fn, name = ((lib.sfb_attn_split_grad, "sfb_attn_split_grad") if cls
                else (lib.sfb_attn_split_grad_nocls, "sfb_attn_split_grad_nocls"))
    L.check(fn(dmerged.data_ptr(), b, heads, nq, hd, int(residual), do.hi_ptr(), do.lo_ptr(), dq.data_ptr(), _stream()),
            name)
    _count()


def _tokpool_desc(b, c, thw, othw, kernel, stride, cls):
    d = L.TokPoolDesc()
    d.b, d.c = b, c
    d.t, d.h, d.w = thw
    d.ot, d.oh, d.ow = othw
    d.kt, d.kh, d.kw = kernel
    d.st, d.sh, d.sw = stride
    d.no_cls = 0 if cls else 1
    return d


def token_maxpool_fwd(x: torch.Tensor, b: int, c: int, thw, othw, kernel, stride, out: torch.Tensor,
                      argmax: torch.Tensor, cls: bool = True) -> None:
    """MaxPool3d(kernel, stride, padding kernel // 2) over the token grid of x [b, cls + thw, c]; the cls row passes
    through; argmax (uint8 tap) is kept for the backward."""
    d = _tokpool_desc(b, c, thw, othw, kernel, stride, cls)
    d.x, d.out, d.argmax = x.data_ptr(), out.data_ptr(), argmax.data_ptr()
    L.check(L.load().sfb_token_maxpool_fwd(C.byref(d), _stream()), "sfb_token_maxpool_fwd")
    _count()


def token_maxpool_bwd(dout: torch.Tensor, argmax: torch.Tensor, b: int, c: int, thw, othw, kernel, stride,
                      dx: torch.Tensor, cls: bool = True) -> None:
    d = _tokpool_desc(b, c, thw, othw, kernel, stride, cls)
    d.argmax = argmax.data_ptr()
    d.dout, d.dx, d.dx_accumulate = dout.data_ptr(), dx.data_ptr(), 0
    L.check(L.load().sfb_token_maxpool_bwd(C.byref(d), _stream()), "sfb_token_maxpool_bwd")
    _count()


def residual_add(src: torch.Tensor, src_bias, y: torch.Tensor, y_bias, scale, rows: int, c: int, tokens: int,
                 out: torch.Tensor) -> None:
    """out[rows, c] = (src + src_bias) + scale[row // tokens] * (y + y_bias): a block's residual with stochastic depth
    (``scale`` None: 1)."""
    L.check(L.load().sfb_residual_add(src.data_ptr(), _ptr(src_bias), y.data_ptr(), y_bias.data_ptr(), _ptr(scale), rows,
                                      c, tokens, out.data_ptr(), _stream()), "sfb_residual_add")
    _count()


def bias_gelu(y: torch.Tensor, bias, rows: int, c: int, out: Planes) -> None:
    """planes[rows, c] = GELU(y + bias) (the exact erf form)."""
    assert out.rows == rows and out.c == c and out.pitch == c
    L.check(L.load().sfb_bias_gelu(y.data_ptr(), bias.data_ptr(), rows, c, out.hi_ptr(), out.lo_ptr(), _stream()),
            "sfb_bias_gelu")
    _count()


def bias_gelu_bwd(dh: torch.Tensor, y: torch.Tensor, bias, rows: int, c: int, dpre: Planes,
                  dpre_f32: torch.Tensor) -> None:
    """Gradient w.r.t. y + bias of ``bias_gelu`` -> planes and fp32 [rows, c]."""
    assert dpre.rows == rows and dpre.c == c and dpre.pitch == c
    L.check(L.load().sfb_bias_gelu_bwd(dh.data_ptr(), y.data_ptr(), bias.data_ptr(), rows, c, dpre.hi_ptr(),
                                       dpre.lo_ptr(), dpre_f32.data_ptr(), _stream()), "sfb_bias_gelu_bwd")
    _count()


def scale_split(dx: torch.Tensor, scale, rows: int, c: int, tokens: int, out: Planes, out_f32: torch.Tensor) -> None:
    """out = scale[row // tokens] * dx -> planes and fp32 [rows, c] (``scale`` None: 1)."""
    assert out.rows == rows and out.c == c and out.pitch == c
    L.check(L.load().sfb_scale_split(dx.data_ptr(), _ptr(scale), rows, c, tokens, out.hi_ptr(), out.lo_ptr(),
                                     out_f32.data_ptr(), _stream()), "sfb_scale_split")
    _count()


def droppath_scales(out: torch.Tensor, rates: torch.Tensor, seed: int, step: torch.Tensor) -> None:
    """out[i, j] = per-sample stochastic-depth scale (0 or 1 / keep) of row i's rate for sample j; ``step``: the int64
    device counter mixed into the seed and incremented after use (graph-replay safe)."""
    n, b = out.shape
    assert rates.numel() == n
    L.check(L.load().sfb_droppath_scales(out.data_ptr(), rates.data_ptr(), n, b, seed, step.data_ptr(), _stream()),
            "sfb_droppath_scales")
    _count(2)


# ------------------------------------------------------------------------------------------------ MAE / MaskFeat
def mae_random_masking(noise: torch.Tensor, keep: int, ids_keep: torch.Tensor, ids_restore: torch.Tensor,
                       mask: torch.Tensor, rows: torch.Tensor) -> None:
    """Stable-argsort ranks of noise [b, l] -> ids_keep [b, keep] / ids_restore [b, l] (int32), mask [b, l] and the rows of
    the removed tokens in the [b, 1 + l] decoder sequence (int32)."""
    b, l = noise.shape
    L.check(L.load().sfb_mae_random_masking(noise.data_ptr(), b, l, keep, ids_keep.data_ptr(), ids_restore.data_ptr(),
                                            mask.data_ptr(), rows.data_ptr(), _stream()), "sfb_mae_random_masking")
    _count()


def tokens_assemble_keep(y: torch.Tensor, bias, cls, pos_spatial, pos_temporal, pos_class, ids_keep: torch.Tensor,
                         b: int, keep: int, lt: int, hw: int, e: int, out: torch.Tensor) -> None:
    """``tokens_assemble`` of the kept patches: the separable positions are gathered by ids_keep."""
    L.check(L.load().sfb_tokens_assemble_keep(y.data_ptr(), bias.data_ptr(), cls.data_ptr(), pos_spatial.data_ptr(),
                                              pos_temporal.data_ptr(), pos_class.data_ptr(), ids_keep.data_ptr(), b,
                                              keep, lt, hw, e, out.data_ptr(), _stream()), "sfb_tokens_assemble_keep")
    _count()


def tokens_scatter_keep(dx: torch.Tensor, ids_restore: torch.Tensor, b: int, keep: int, lt: int, e: int,
                        dense: torch.Tensor) -> None:
    """The kept-token gradient [b, 1 + keep, e] scattered onto the dense grid [b, 1 + lt, e] (zero elsewhere)."""
    L.check(L.load().sfb_tokens_scatter_keep(dx.data_ptr(), ids_restore.data_ptr(), b, keep, lt, e, dense.data_ptr(),
                                             _stream()), "sfb_tokens_scatter_keep")
    _count()


def decoder_assemble(z: torch.Tensor, bias, mask_token, pos, ids_restore: torch.Tensor, b: int, keep: int, lt: int,
                     c: int, out: torch.Tensor) -> None:
    """out[b, 1 + lt, c] = the encoder tokens z + bias un-shuffled by ids_restore, mask_token in the removed places, + the
    joint table pos."""
    L.check(L.load().sfb_decoder_assemble(z.data_ptr(), bias.data_ptr(), mask_token.data_ptr(), pos.data_ptr(),
                                          ids_restore.data_ptr(), b, keep, lt, c, out.data_ptr(), _stream()),
            "sfb_decoder_assemble")
    _count()


def decoder_assemble_bwd(dx: torch.Tensor, ids_keep: torch.Tensor, rows: torch.Tensor, b: int, keep: int, lt: int,
                         c: int, dz: torch.Tensor, dpos, dmask, partials: torch.Tensor) -> None:
    """Gradients of ``decoder_assemble``: dz [b, 1 + keep, c], dpos [1 + lt, c], dmask [c].  ``partials``: fp32 scratch of
    at least segment_slabs(1, b * (lt - keep)) * c elements."""
    assert partials.numel() >= segment_slabs(1, b * (lt - keep)) * c
    L.check(L.load().sfb_decoder_assemble_bwd(dx.data_ptr(), ids_keep.data_ptr(), rows.data_ptr(), b, keep, lt, c,
                                              dz.data_ptr(), dpos.data_ptr(), dmask.data_ptr(), partials.data_ptr(),
                                              _stream()), "sfb_decoder_assemble_bwd")
    _count(4)


def rows_gather(src: torch.Tensor, src_pitch: int, rows: Optional[torch.Tensor], n: int, c: int, bias,
                out: torch.Tensor) -> None:
    """out[n, c] = src[rows[i], :c] (+ bias); a null ``rows`` takes rows 0 .. n - 1."""
    L.check(L.load().sfb_rows_gather(src.data_ptr(), src_pitch, _ptr(rows), n, c, _ptr(bias), out.data_ptr(),
                                     _stream()), "sfb_rows_gather")
    _count()


def rows_scatter(src: torch.Tensor, rows: torch.Tensor, n: int, c: int, out: torch.Tensor) -> None:
    """out[rows[i], :c] = src[i] (the other rows untouched)."""
    L.check(L.load().sfb_rows_scatter(src.data_ptr(), rows.data_ptr(), n, c, out.data_ptr(), _stream()),
            "sfb_rows_scatter")
    _count()


def pixel_targets(frames: torch.Tensor, t_stride: int, pred_t: int, patch: int, rows: torch.Tensor, norm: bool,
                  out: torch.Tensor) -> None:
    """The (normalised) pixel labels of the decoder rows ``rows`` of the NCTHW fp32 clip: [len(rows), pred_t * p * p * C]."""
    b, c, t, h, w = frames.shape
    assert frames.dtype == F32 and frames.is_contiguous()
    L.check(L.load().sfb_pixel_targets(frames.data_ptr(), b, c, t, h, w, t_stride, pred_t, patch, rows.data_ptr(),
                                       rows.numel(), int(norm), out.data_ptr(), _stream()), "sfb_pixel_targets")
    _count()


def hog_targets(frames: torch.Tensor, t_stride: int, nbins: int, cell: int, fs: int, out: torch.Tensor) -> None:
    """HOG regression targets of every output token of the NCTHW fp32 clip: [b, (t / t_stride) * fs * fs, ...]."""
    b, c, t, h, w = frames.shape
    assert frames.dtype == F32 and frames.is_contiguous()
    L.check(L.load().sfb_hog_targets(frames.data_ptr(), b, c, t, h, w, t_stride, nbins, cell, fs, out.data_ptr(),
                                     _stream()), "sfb_hog_targets")
    _count()


def mask_upsample(fmask: torch.Tensor, thw, out: torch.Tensor) -> None:
    """The cube mask [b, mt, mh, mw] at the token grid thw: out [b, t * h * w]."""
    b, mt, mh, mw = fmask.shape
    L.check(L.load().sfb_mask_upsample(fmask.data_ptr(), b, mt, mh, mw, *thw, out.data_ptr(), _stream()),
            "sfb_mask_upsample")
    _count()


def tokens_assemble_masked(y: torch.Tensor, bias, cls, mask_token, tokmask: torch.Tensor, b: int, lt: int, e: int,
                           out: torch.Tensor) -> None:
    """out = [cls ; y + bias] with mask_token in place of the masked tokens (tokmask [b, lt])."""
    L.check(L.load().sfb_tokens_assemble_masked(y.data_ptr(), bias.data_ptr(), cls.data_ptr(), mask_token.data_ptr(),
                                                tokmask.data_ptr(), b, lt, e, out.data_ptr(), _stream()),
            "sfb_tokens_assemble_masked")
    _count()


def tokens_split_grad_masked(dx: torch.Tensor, tokmask: torch.Tensor, b: int, lt: int, e: int, dy: Planes,
                             dy_f32: torch.Tensor, dmasked: torch.Tensor) -> None:
    """``tokens_split_grad`` of ``tokens_assemble_masked``: the masked tokens' gradient goes to dmasked [b * lt, e]."""
    assert dy.rows == b * lt and dy.c == e and dy.pitch == e
    L.check(L.load().sfb_tokens_split_grad_masked(dx.data_ptr(), tokmask.data_ptr(), b, lt, e, dy.hi_ptr(), dy.lo_ptr(),
                                                  dy_f32.data_ptr(), dmasked.data_ptr(), _stream()),
            "sfb_tokens_split_grad_masked")
    _count()


def rows_unpad_bias(y: torch.Tensor, y_pitch: int, bias, b: int, n: int, c: int, out: torch.Tensor) -> None:
    """out[b, n, c] = y[b, 1 + i, :c] + bias: the prediction rows without the cls row."""
    L.check(L.load().sfb_rows_unpad_bias(y.data_ptr(), y_pitch, bias.data_ptr(), b, n, c, out.data_ptr(), _stream()),
            "sfb_rows_unpad_bias")
    _count()


def rows_pad_split(src: torch.Tensor, b: int, n: int, c: int, out: Planes) -> None:
    """The backward of ``rows_unpad_bias``: src [b, n, c] -> planes [b * (1 + n), out.c] (cls rows and pad columns
    zero)."""
    assert out.rows == b * (n + 1) and out.pitch == out.c >= c
    L.check(L.load().sfb_rows_pad_split(src.data_ptr(), b, n, c, out.c, out.hi_ptr(), out.lo_ptr(), _stream()),
            "sfb_rows_pad_split")
    _count()
