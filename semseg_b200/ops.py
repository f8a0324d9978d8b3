"""Tensor-level wrappers over the C-ABI (semseg_b200/_lib.py): every function takes CUDA tensors,
launches on torch's current stream and returns tensors. PyTorch is used for device memory and streams
only; the arithmetic happens in libsemseg_b200.so. No function here has a CPU or eager fallback.
"""
import ctypes

import torch

from . import _lib
from . import p2p
from ._lib import ConvDesc, WgradDesc, EPI_RAW, EPI_AFFINE, EPI_F32, MAX_TAPS


# bf16x3: K blocks (64-channel block x tap) one tensor-core accumulation chain may span (8 x 4 x 3 = 96 MMA steps; the
# truncating fp32 accumulation of the tensor core loses ~2^-24 per step towards zero, tools/probe_accum.py)
X3_MAX_KBLOCKS = 8

_raw_stream = getattr(torch._C, "_cuda_getCurrentRawStream", None)
_cur_device = getattr(torch._C, "_cuda_getDevice", None)


def _stream():
    """torch's current CUDA stream of the current device as a raw cudaStream_t. Called once per kernel launch (~700
    times per training step), so it goes through the two C accessors instead of building a torch.cuda.Stream object
    (which was a quarter of the host-side step time, tools/profile_cpu.py)."""
    if _raw_stream is not None and _cur_device is not None:
        return ctypes.c_void_p(_raw_stream(_cur_device()))
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _require_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise _lib.SemsegError("semseg_b200 ops require CUDA tensors (no CPU fallback); got device %s" % t.device)


# ------------------------------------------------------------------------------------------------ activation storage
# An activation is either a plain bf16 NHWC tensor [N,H,W,C] ("bf16", the speed configuration) or a SPLIT tensor
# [2,N,H,W,C]: plane 0 = hi = bf16(v), plane 1 = lo = bf16(v - hi) (16 mantissa bits, csrc/act.cuh). The conv kernels
# consume split operands as three K segments (bf16x3); every other kernel reads hi + lo and re-splits its result. The
# storage form is chosen once per model call (precision.py) and every op follows the form of its input.
def is_split(t):
    return t is not None and t.dim() == 5


def _nhwc_meta(t):
    """(N, H, W, C, pitch) of a bf16 NHWC activation (plain 4-D or split 5-D) whose channel dim may be a slice of a
    wider buffer."""
    assert t.dtype == torch.bfloat16 and t.dim() in (4, 5), (t.shape, t.dtype)
    if t.dim() == 5:
        assert t.shape[0] == 2, "split activation must be [2,N,H,W,C] (hi, lo planes)"
    n, h, w, c = t.shape[-4:]
    sn, sh, sw, sc = t.stride()[-4:]
    assert sc == 1 and sh == sw * w and sn == sh * h, "NHWC tensor must be pixel-contiguous (stride %s)" % (t.stride(),)
    return n, h, w, c, sw


def _lo(t):
    """Pointer to the lo plane of a split activation, NULL for a plain one."""
    if t is not None and t.dim() == 5:
        return ctypes.c_void_p(t.data_ptr() + 2 * t.stride(0))
    return ctypes.c_void_p(0)


def _lo_int(t):
    return t.data_ptr() + 2 * t.stride(0) if (t is not None and t.dim() == 5) else 0


def empty_act(shape, split, device):
    """Uninitialised activation of NHWC shape `shape` in the requested storage form."""
    return torch.empty(((2,) + tuple(shape)) if split else tuple(shape), dtype=torch.bfloat16, device=device)


def _same_form(*ts):
    forms = {t.dim() == 5 for t in ts if t is not None}
    assert len(forms) <= 1, "activations of one call must all be plain or all be split"


def act_batch_slice(t, a, b):
    """Images a..b of an activation (either storage form)."""
    return t[:, a:b] if t.dim() == 5 else t[a:b]


def round_up(a, b):
    return (a + b - 1) // b * b


# ------------------------------------------------------------------------------------------------ psa mask
def psamask_fwd(x, psa_type, mask_h, mask_w):
    _require_cuda(x)
    lib = _lib.load()
    assert x.dtype == torch.float32 and x.is_contiguous()
    n, c, h, w = x.shape
    out = torch.empty((n, h * w, h, w), dtype=torch.float32, device=x.device)
    _lib.check(lib.semseg_psamask_fwd(psa_type, _ptr(x), _ptr(out), n, h, w, mask_h, mask_w, _stream()),
               "semseg_psamask_fwd")
    return out


def psamask_bwd(grad_out, psa_type, mask_h, mask_w):
    _require_cuda(grad_out)
    lib = _lib.load()
    assert grad_out.dtype == torch.float32 and grad_out.is_contiguous()
    n, hw, h, w = grad_out.shape
    din = torch.empty((n, mask_h * mask_w, h, w), dtype=torch.float32, device=grad_out.device)
    _lib.check(lib.semseg_psamask_bwd(psa_type, _ptr(grad_out), _ptr(din), n, h, w, mask_h, mask_w, _stream()),
               "semseg_psamask_bwd")
    return din


# ------------------------------------------------------------------------------------------------ fused PSA attention
def _psa_form(compact, softmax):
    return (_lib.PSA_DENSE if compact else 0) | (0 if softmax else _lib.PSA_NO_SOFTMAX)


def psa_attend(attn, feat, psa_type, mask_h, mask_w, scale, stats=None, mode=0, compact=False, softmax=True):
    """mode 0: (out, stats) = fused mask-gather -> softmax -> aggregation (model/psanet.py:81-91) of the fp32 NHWC logits
    `attn` [N,h,w,>=mask_h*mask_w] and the NHWC activation `feat` [N,h,w,512]; mode 1: the feature gradient (pass dout as
    `feat` and the forward's `stats`). compact: the dense mask form (mask_h*mask_w == h*w, model/psanet.py:76-79);
    softmax=False: P = the gathered logits, and stats is None."""
    _require_cuda(attn, feat)
    lib = _lib.load()
    assert attn.dtype == torch.float32 and attn.dim() == 4 and attn.is_contiguous()
    n, h, w, c, fp = _nhwc_meta(feat)
    assert tuple(attn.shape[:3]) == (n, h, w) and attn.shape[3] >= mask_h * mask_w
    out = empty_act((n, h, w, c), is_split(feat), feat.device)
    if stats is None and softmax:
        assert mode == 0
        stats = torch.empty((n, h * w, 2), dtype=torch.float32, device=feat.device)
    _lib.check(lib.semseg_psa_attend_ex(mode, psa_type, _psa_form(compact, softmax), _ptr(attn), attn.shape[3], _ptr(feat),
                                        _lo(feat), fp, _ptr(stats), _ptr(out), _lo(out), c, n, h, w, mask_h, mask_w, c,
                                        float(scale), _stream()),
               "semseg_psa_attend")
    return out, stats


def psa_attend_bwd_attn(attn, stats, feat, out, dout, psa_type, mask_h, mask_w, scale, compact=False, softmax=True):
    """Gradient of psa_attend w.r.t. the attention logits (same shape as attn, zero outside the mask windows). Without
    softmax, stats and out are not read and may be None."""
    lib = _lib.load()
    n, h, w, c, fp = _nhwc_meta(feat)
    op, dp = (_nhwc_meta(out)[4] if out is not None else c), _nhwc_meta(dout)[4]
    _same_form(feat, out, dout)
    dattn = torch.empty_like(attn)
    _lib.check(lib.semseg_psa_attend_bwd_attn_ex(psa_type, _psa_form(compact, softmax), _ptr(attn), attn.shape[3],
                                                 _ptr(stats), _ptr(feat), _lo(feat), fp, _ptr(out), _lo(out), op,
                                                 _ptr(dout), _lo(dout), dp, _ptr(dattn), n, h, w, mask_h, mask_w, c,
                                                 float(scale), _stream()),
               "semseg_psa_attend_bwd_attn")
    return dattn


# ------------------------------------------------------------------------------------------------ weights
class PackedWeight:
    """bf16 operand slabs of one conv weight: wf [taps][Cout][Cin_p] (fprop), wd [taps][Cin][Cout_p] (dgrad) or None,
    wp [1][Cout][32] or None (the stem conv as a 1x1 conv over im2col3x3s2 patches: column t*Cin + c holds tap t of
    input channel c); with split=True each is [2][...] = the hi slab followed by the lo slab (bf16x3 operand mode)."""
    __slots__ = ("wf", "wd", "wp", "cout", "cin", "taps", "ksize", "split")

    def __init__(self, wf, wd, wp, cout, cin, taps, ksize, split=False):
        self.wf, self.wd, self.wp = wf, wd, wp
        self.cout, self.cin, self.taps, self.ksize, self.split = cout, cin, taps, ksize, split


def _slab(taps, rows, cols, split, device):
    return torch.empty(((2,) if split else ()) + (taps, rows, cols), dtype=torch.bfloat16, device=device)


def pack_weights(w, need_dgrad=True, split=False):
    """w: fp32 OIHW parameter -> PackedWeight (a one-conv WeightPackPlan, packed once)."""
    w = w.detach()
    plan = WeightPackPlan([w if w.is_contiguous() else w.contiguous()], split, dgrad=need_dgrad)
    plan.refresh()
    return plan.packs[0]


class WeightPackPlan:
    """Persistent bf16 operand slabs for a list of conv weights, refreshed in ONE launch (semseg_pack_weights_multi).

    The fp32 OIHW parameters stay the masters (optimizer / DDP / checkpoints); after an optimizer step every conv of the
    model needs new slabs. The plan owns the slabs of every conv (wf; wd when `dgrad`; wp where `patches[k]`) and a
    device-side item table; `refresh()` re-packs all of them into the same buffers. Building a plan uploads the table,
    so it cannot be done while a CUDA graph is being captured; refreshing can."""

    def __init__(self, weights, split=False, dgrad=True, patches=None):
        _require_cuda(*weights)
        self.split = bool(split)
        self.weights = [w for w in weights]
        self.ptrs = [w.data_ptr() for w in weights]
        self.packs = []
        items = (_lib.PackItem * len(weights))()
        tile0, max_taps = 0, 1
        for k, w in enumerate(weights):
            assert w.dtype == torch.float32 and w.dim() == 4 and w.is_contiguous() and w.shape[2] == w.shape[3]
            cout, cin, kh, _ = w.shape
            taps = kh * kh
            patch = bool(patches and patches[k])
            assert taps <= MAX_TAPS and (not patch or (taps == 9 and cin <= 3))
            cin_p, cout_p = round_up(cin, 8), round_up(cout, 8)
            wf = _slab(taps, cout, cin_p, self.split, w.device)
            wd = _slab(taps, cin, cout_p, self.split, w.device) if dgrad else None
            wp = _slab(1, cout, 32, self.split, w.device) if patch else None
            self.packs.append(PackedWeight(wf, wd, wp, cout, cin, taps, kh, self.split))
            it = items[k]
            it.w, it.wf, it.wd, it.wp = w.data_ptr(), wf.data_ptr(), _ptr(wd).value, _ptr(wp).value
            it.Cout, it.Cin, it.taps, it.cols_f, it.cols_d = cout, cin, taps, cin_p, cout_p
            it.tile0, it.tiles_ci, it.split = tile0, (cin_p + 31) // 32, int(self.split)
            tile0 += it.tiles_ci * ((cout_p + 31) // 32)
            max_taps = max(max_taps, taps)
        self.n_items, self.n_tiles, self.max_taps = len(weights), tile0, max_taps
        raw = torch.frombuffer(bytearray(bytes(items)), dtype=torch.uint8)
        self.items_dev = raw.to(weights[0].device)

    def valid_for(self, weights, split=False):
        return (bool(split) == self.split and len(weights) == len(self.ptrs) and
                all(w.data_ptr() == p for w, p in zip(weights, self.ptrs)))

    def refresh(self):
        lib = _lib.load()
        _lib.check(lib.semseg_pack_weights_multi(_ptr(self.items_dev), self.n_items, self.n_tiles, self.max_taps,
                                                 _stream()), "semseg_pack_weights_multi")


def conv_taps(ksize, dilation, transpose=False):
    """[(dh, dw, wtap)] of a stride-1 'same' conv; transpose=True gives the dgrad taps."""
    taps = []
    half = ksize // 2
    for r in range(ksize):
        for s in range(ksize):
            dh, dw = (r - half) * dilation, (s - half) * dilation
            if transpose:
                dh, dw = -dh, -dw
            taps.append((dh, dw, r * ksize + s))
    return taps


def _fill_taps(desc, taps, with_wtap=True, img_add=None):
    assert 1 <= len(taps) <= MAX_TAPS
    desc.taps = len(taps)
    for i, t in enumerate(taps):
        desc.dh[i], desc.dw[i] = t[0], t[1]
        if with_wtap:
            desc.wtap[i] = t[2]
        desc.img_add[i] = img_add[i] if img_add is not None else 0
    desc.img_mul = 1


def conv_taps_s2(ksize, n):
    """Taps of a stride-2 'same' conv (k in {1,3}) on the 2x2 phase tensor [4N,Hh,Wh,C] (space_to_phases):
    [(dh, dw, wtap, img_add, (ph, pw))]: input row 2*ho + r - k//2 lives in phase (r+1)&1 at row ho + dh."""
    taps = []
    for r in range(ksize):
        for s in range(ksize):
            if ksize == 3:
                ph, dh = (0, 0) if r == 1 else (1, -1 if r == 0 else 0)
                pw, dw = (0, 0) if s == 1 else (1, -1 if s == 0 else 0)
            else:
                ph = pw = dh = dw = 0
            taps.append((dh, dw, r * ksize + s, (ph * 2 + pw) * n, (ph, pw)))
    return taps


def _planes(*ts):
    """[(plane views...)] of activations that share a storage form: one tuple for plain tensors, two for split."""
    _same_form(*ts)
    if ts[0].dim() == 5:
        return [tuple(t[0] for t in ts), tuple(t[1] for t in ts)]
    return [tuple(ts)]


def im2col3x3s2(x, cin):
    """NHWC bf16 x (first `cin` <= 3 channels real) -> patches [N, Ho, Wo, 32] of the 3x3 / stride 2 / pad 1 stem conv."""
    lib = _lib.load()
    n, h, w, _, p = _nhwc_meta(x)
    out = empty_act((n, (h - 1) // 2 + 1, (w - 1) // 2 + 1, 32), is_split(x), x.device)
    for xi, oi in _planes(x, out):      # pure data movement: the hi and lo planes are gathered independently
        _lib.check(lib.semseg_im2col3x3s2(_ptr(xi), p, n, h, w, int(cin), _ptr(oi), _stream()), "semseg_im2col3x3s2")
    return out


def stem_dgrad3x3s2(dy, wp, cin, h, w):
    """Input gradient of the stem conv (3x3 / stride 2 / pad 1, `cin` <= 3 channels) as fp32 NCHW [N, cin, h, w], from
    the conv output's gradient `dy` (activation [N, Ho, Wo, 64], either storage form) and the patch slab `wp` of
    PackedWeight (split exactly when dy is: bf16x3)."""
    _require_cuda(dy, wp)
    lib = _lib.load()
    n, ho, wo, cout, p = _nhwc_meta(dy)
    split = is_split(dy)
    assert wp.dtype == torch.bfloat16 and wp.is_contiguous() and wp.dim() == (4 if split else 3), \
        "the patch slab must be [1][Cout][32] (plain) or [2][1][Cout][32] (split), in dy's storage form"
    dx = torch.empty((n, cin, h, w), dtype=torch.float32, device=dy.device)
    _lib.check(lib.semseg_stem_dgrad3x3s2(_ptr(dy), _lo(dy), p, n, ho, wo, h, w, int(cin), cout, _ptr(wp), int(split),
                                          _ptr(dx), _stream()), "semseg_stem_dgrad3x3s2")
    return dx


def space_to_phases(x):
    """x [N,H,W,C] bf16 -> [4N, (H+1)//2, (W+1)//2, C] (phase-major)."""
    _require_cuda(x)
    lib = _lib.load()
    n, h, w, c, p = _nhwc_meta(x)
    xp = empty_act((4 * n, (h + 1) // 2, (w + 1) // 2, c), is_split(x), x.device)
    for xi, oi in _planes(x, xp):
        _lib.check(lib.semseg_space_to_phases(_ptr(xi), p, n, h, w, c, _ptr(oi), _stream()), "semseg_space_to_phases")
    return xp


def phases_to_space(xp, n, h, w):
    lib = _lib.load()
    c = xp.shape[-1]
    assert xp.is_contiguous() and xp.shape[-4] == 4 * n
    x = empty_act((n, h, w, c), is_split(xp), xp.device)
    for xi, oi in _planes(xp, x):
        _lib.check(lib.semseg_phases_to_space(_ptr(xi), n, h, w, c, _ptr(oi), _stream()), "semseg_phases_to_space")
    return x


# ------------------------------------------------------------------------------------------------ conv
def conv_stats_rows(n, h, w, cout):
    return int(_lib.load().semseg_conv_stats_rows(n, h, w, cout))


def conv_fprop(x, w3d, cout, taps, *, out=None, epi=EPI_RAW, relu=False, scale=None, shift=None, residual=None,
               stats=False, out_f32=None, img_add=None, out_nhw=None):
    """Implicit-GEMM conv of NHWC bf16 `x` with packed weights `w3d` [n_wtaps][rows][cols].

    Returns (y, stats_partial); y is bf16 NHWC [N,H,W,cout] (or the fp32 tensor in F32 mode); stats_partial is the
    per-CTA [rows][3][cout] (sum, sum of squares, count) buffer when stats=True.
    """
    _require_cuda(x, w3d)
    lib = _lib.load()
    nin, hin, win, cin, xp = _nhwc_meta(x)
    split = is_split(x)
    n, h, w = out_nhw if out_nhw is not None else (nin, hin, win)   # output pixel grid (differs for phase tensors)
    d = ConvDesc()
    d.N, d.H, d.W, d.Cin, d.Cout = n, h, w, cin, cout
    d.x, d.Nin, d.Hin, d.Win, d.x_pitch = x.data_ptr(), nin, hin, win, xp
    d.x_lo = _lo_int(x)
    assert w3d.dtype == torch.bfloat16 and w3d.is_contiguous() and w3d.dim() == (4 if split else 3), \
        "packed weights must be [taps][rows][cols] (plain) or [2][taps][rows][cols] (split, hi then lo slab)"
    d.w, d.n_wtaps, d.w_rows, d.w_cols = w3d.data_ptr(), w3d.shape[-3], w3d.shape[-2], w3d.shape[-1]
    d.w_split = int(split)
    _fill_taps(d, taps, img_add=img_add)
    d.epi_mode, d.relu = epi, int(bool(relu))
    sp = None
    if epi == EPI_F32:
        if out_f32 is None:
            out_f32 = torch.empty((n, h, w, cout), dtype=torch.float32, device=x.device)
        assert out_f32.dtype == torch.float32 and out_f32.stride(-1) == 1
        d.out_f32, d.out_pitch = out_f32.data_ptr(), out_f32.stride(2)
        y = out_f32
    else:
        if out is None:
            out = empty_act((n, h, w, cout), split, x.device)
        on, oh, ow, oc, op = _nhwc_meta(out)
        assert (on, oh, ow, oc) == (n, h, w, cout) and is_split(out) == split
        d.y, d.y_pitch, d.y_lo = out.data_ptr(), op, _lo_int(out)
        y = out
    if scale is not None:
        assert scale.dtype == torch.float32 and scale.numel() >= cout
        d.scale = scale.data_ptr()
    if shift is not None:
        assert shift.dtype == torch.float32 and shift.numel() >= cout
        d.shift = shift.data_ptr()
    if residual is not None:
        rn, rh, rw, rc, rp = _nhwc_meta(residual)
        assert (rn, rh, rw, rc) == (n, h, w, cout) and is_split(residual) == split
        d.residual, d.res_pitch, d.residual_lo = residual.data_ptr(), rp, _lo_int(residual)
    # bf16x3: convs with long K are K-sliced (fp32 partials summed round-to-nearest by conv_splitk_finish), because one
    # tensor-core accumulation chain loses ~2^-24 per MMA step towards zero (tools/probe_accum.py)
    k_slices = int(lib.semseg_conv_k_slices(cin, len(taps), X3_MAX_KBLOCKS)) if (split and epi != EPI_F32) else 1
    if k_slices > 1:
        part = torch.empty((k_slices, n, h, w, cout), dtype=torch.float32, device=x.device)
        d.epi_mode, d.relu = EPI_F32, 0
        d.out_f32, d.out_pitch = part.data_ptr(), cout
        d.k_slices, d.slice_stride = k_slices, part.stride(0)
        sc, sh, rs, rsl, rpitch, ylo = d.scale, d.shift, d.residual, d.residual_lo, d.res_pitch, d.y_lo
        d.scale = d.shift = d.residual = d.residual_lo = d.y_lo = None
        _lib.check(lib.semseg_conv_fprop(ctypes.byref(d), _stream()), "semseg_conv_fprop (K-sliced)")
        m = n * h * w
        if stats:
            assert epi == EPI_RAW
            sp = torch.empty((int(lib.semseg_conv_splitk_rows(m)), 3, cout), dtype=torch.float32, device=x.device)
        _lib.check(lib.semseg_conv_splitk_finish(_ptr(part), k_slices, part.stride(0), cout, m, cout, epi,
                                                 int(bool(relu)), sc, sh, rs, rsl, rpitch, d.y, ylo, d.y_pitch,
                                                 _ptr(sp), _stream()), "semseg_conv_splitk_finish")
        return y, sp
    if stats:
        assert epi == EPI_RAW
        sp = torch.empty((conv_stats_rows(n, h, w, cout), 3, cout), dtype=torch.float32, device=x.device)
        d.stats_partial = sp.data_ptr()
    _lib.check(lib.semseg_conv_fprop(ctypes.byref(d), _stream()), "semseg_conv_fprop")
    return y, sp


def conv_wgrad(x, dy, cin, cout, taps, grad_out=None, accumulate=False, img_add=None):
    """dW (fp32 OIHW [cout][cin][k][k]) from NHWC bf16 x and dy. The pixel grid is dy's; `x` may be a phase tensor
    (stride-2 convs) addressed through `img_add`."""
    _require_cuda(x, dy)
    lib = _lib.load()
    nin, hin, win, xc, xp = _nhwc_meta(x)
    n, h, w, dc, dp = _nhwc_meta(dy)
    assert xc >= cin and dc >= cout
    assert img_add is not None or (nin, hin, win) == (n, h, w)
    _same_form(x, dy)
    d = WgradDesc()
    d.N, d.H, d.W, d.Cin, d.Cout = n, h, w, cin, cout
    d.x, d.Nin, d.Hin, d.Win, d.x_pitch = x.data_ptr(), nin, hin, win, xp
    d.dy, d.dy_pitch = dy.data_ptr(), dp
    d.x_lo, d.dy_lo = _lo_int(x), _lo_int(dy)
    _fill_taps(d, taps, with_wtap=False, img_add=img_add)
    d.n_splits = 0
    splits = lib.semseg_conv_wgrad_splits(ctypes.byref(d))
    if splits <= 0:
        raise _lib.SemsegError("semseg_conv_wgrad_splits failed (%d)" % splits)
    ntaps = len(taps)
    part = torch.empty((splits, ntaps, cout, cin), dtype=torch.float32, device=x.device)
    d.dw_partial = part.data_ptr()
    d.n_splits = splits
    _lib.check(lib.semseg_conv_wgrad(ctypes.byref(d), _stream()), "semseg_conv_wgrad")
    k = int(round(ntaps ** 0.5))
    if grad_out is None:
        grad_out = torch.empty((cout, cin, k, k), dtype=torch.float32, device=x.device)
        accumulate = False
    assert grad_out.is_contiguous() and grad_out.dtype == torch.float32
    _lib.check(lib.semseg_wgrad_reduce(_ptr(part), splits, ntaps, cout, cin, _ptr(grad_out), int(accumulate),
                                       _stream()), "semseg_wgrad_reduce")
    return grad_out


# ------------------------------------------------------------------------------------------------ layout
def nchw_to_nhwc_bf16(x, pad_to=8, split=False):
    _require_cuda(x)
    lib = _lib.load()
    assert x.dtype == torch.float32 and x.is_contiguous()
    n, c, h, w = x.shape
    cp = round_up(c, pad_to)
    shape = ((2,) if split else ()) + (n, h, w, cp)
    out = (torch.zeros if cp != c else torch.empty)(shape, dtype=torch.bfloat16, device=x.device)
    _lib.check(lib.semseg_nchw_f32_to_nhwc_bf16(_ptr(x), _ptr(out), _lo(out), n, c, h, w, cp, _stream()),
               "semseg_nchw_f32_to_nhwc_bf16")
    return out


def nhwc_bf16_to_nchw(x):
    _require_cuda(x)
    lib = _lib.load()
    n, h, w, c, p = _nhwc_meta(x)
    out = torch.empty((n, c, h, w), dtype=torch.float32, device=x.device)
    _lib.check(lib.semseg_nhwc_bf16_to_nchw_f32(_ptr(x), _lo(x), _ptr(out), n, c, h, w, p, _stream()),
               "semseg_nhwc_bf16_to_nchw_f32")
    return out


def nhwc_f32_to_nchw(x):
    _require_cuda(x)
    lib = _lib.load()
    assert x.dtype == torch.float32 and x.dim() == 4 and x.stride(-1) == 1
    n, h, w, c = x.shape
    out = torch.empty((n, c, h, w), dtype=torch.float32, device=x.device)
    _lib.check(lib.semseg_nhwc_f32_to_nchw_f32(_ptr(x), _ptr(out), n, c, h, w, x.stride(2), _stream()),
               "semseg_nhwc_f32_to_nchw_f32")
    return out


# ------------------------------------------------------------------------------------------------ batch norm
def bn_workspace(m, c, device):
    nf = int(_lib.load().semseg_bn_workspace_floats(m, c))
    return torch.empty((nf,), dtype=torch.float32, device=device), nf


def bn_merge_partials(stats_partial):
    lib = _lib.load()
    t, _, c = stats_partial.shape
    out = torch.empty((3, c), dtype=torch.float32, device=stats_partial.device)
    _lib.check(lib.semseg_bn_merge_partials(_ptr(stats_partial), t, c, _ptr(out), _stream()),
               "semseg_bn_merge_partials")
    return out


def bn_finalize(rank_stats, gamma, beta, eps, momentum, running_mean, running_var):
    """rank_stats [R][3][C] -> (mean_invstd [2][C], scale_shift [2][C]); updates running stats in place."""
    lib = _lib.load()
    if rank_stats.dim() == 2:
        rank_stats = rank_stats.unsqueeze(0)
    r, _, c = rank_stats.shape
    assert rank_stats.is_contiguous()
    mi = torch.empty((3, c), dtype=torch.float32, device=rank_stats.device)      # mean, invstd, total count
    ss = torch.empty((2, c), dtype=torch.float32, device=rank_stats.device)
    _lib.check(lib.semseg_bn_finalize(_ptr(rank_stats), r, c, _ptr(gamma), _ptr(beta), float(eps), float(momentum),
                                      _ptr(running_mean), _ptr(running_var), _ptr(mi), _ptr(ss), _stream()),
               "semseg_bn_finalize")
    return mi, ss


def _peer_args(px):
    """(peer_bufs, world, rank, slot, slot_floats, seq_ptr) of the statistics entry points: the next exchange of the
    NVLink peer exchange `px` (p2p.PeerExchange), or a single rank (NULL peer table) when `px` is None."""
    if px is None:
        return None, 1, 0, 0, 0, None
    return px.data_ptrs, px.world, px.rank, px.next(), p2p.SLOT_FLOATS, _ptr(px.step)


def bn_finalize_partials(stats_partial, gamma, beta, eps, momentum, running_mean, running_var, px=None):
    """Per-tile conv partials -> (mean_invstd, scale_shift) in one launch; with `px` the statistics of every rank, exchanged
    inside the kernel over peer memory (SyncBN)."""
    lib = _lib.load()
    t, _, c = stats_partial.shape
    buf = torch.empty((5, c), dtype=torch.float32, device=stats_partial.device)
    mi, ss = buf[:3], buf[3:]                               # (mean, invstd, total count), (scale, shift)
    _lib.check(lib.semseg_bn_finalize_partials(_ptr(stats_partial), t, c, _ptr(gamma), _ptr(beta),
                                               float(eps), float(momentum), _ptr(running_mean), _ptr(running_var),
                                               _ptr(mi), _ptr(ss), *_peer_args(px), _stream()),
               "semseg_bn_finalize_partials")
    return mi, ss


def bn_fold_eval(gamma, beta, running_mean, running_var, eps):
    lib = _lib.load()
    c = running_mean.numel()
    ss = torch.empty((2, c), dtype=torch.float32, device=running_mean.device)
    _lib.check(lib.semseg_bn_fold_eval(_ptr(gamma), _ptr(beta), _ptr(running_mean), _ptr(running_var), float(eps), c,
                                       _ptr(ss), _stream()), "semseg_bn_fold_eval")
    return ss


def bn_apply(x, scale_shift, residual=None, relu=True, out=None):
    _require_cuda(x)
    lib = _lib.load()
    n, h, w, c, xp = _nhwc_meta(x)
    if out is None:
        out = empty_act((n, h, w, c), is_split(x), x.device)
    _, _, _, oc, op = _nhwc_meta(out)
    assert oc == c
    rp = 0
    if residual is not None:
        _, _, _, rc, rp = _nhwc_meta(residual)
        assert rc == c
    _same_form(x, out, residual)
    _lib.check(lib.semseg_bn_apply(_ptr(x), _lo(x), xp, _ptr(scale_shift), _ptr(residual), _lo(residual), rp,
                                   _ptr(out), _lo(out), op, n * h * w, c, int(bool(relu)), _stream()),
               "semseg_bn_apply")
    return out


def bn_bwd_reduce(dy, y, x, mean_invstd, relu, scale_shift=None, px=None):
    """-> (sums_local [2][C], sums_total [2][C]) = (sum dz, sum dz*xhat) of this rank and over all ranks, added inside
    the kernel over peer memory when `px` is given; without `px` both are the same tensor."""
    lib = _lib.load()
    n, h, w, c, dp = _nhwc_meta(dy)
    _, _, _, _, xp = _nhwc_meta(x)
    yp = _nhwc_meta(y)[4] if y is not None else 0
    m = n * h * w
    ws, nf = bn_workspace(m, c, dy.device)
    out = torch.empty((2 if px is not None else 1, 2, c), dtype=torch.float32, device=dy.device)
    local, total = out[0], out[-1]
    _same_form(dy, y, x)
    _lib.check(lib.semseg_bn_bwd_reduce(_ptr(dy), _lo(dy), dp, _ptr(y), _lo(y), yp, _ptr(x), _lo(x), xp,
                                        _ptr(mean_invstd), _ptr(scale_shift), m, c, int(bool(relu)), _ptr(ws), nf,
                                        _ptr(local), _ptr(total), *_peer_args(px), _stream()),
               "semseg_bn_bwd_reduce")
    return local, total


def bn_bwd_apply(dy, y, x, mean_invstd, gamma, sums, count, relu, want_dres=False, scale_shift=None):
    """Returns (dx bf16, dres bf16 or None, dgamma_dbeta [2][C])."""
    lib = _lib.load()
    n, h, w, c, dp = _nhwc_meta(dy)
    _, _, _, _, xp = _nhwc_meta(x)
    yp = _nhwc_meta(y)[4] if y is not None else 0
    _same_form(dy, y, x)
    split = is_split(dy)
    dx = empty_act((n, h, w, c), split, dy.device)
    dres = empty_act((n, h, w, c), split, dy.device) if want_dres else None
    dgb = torch.empty((2, c), dtype=torch.float32, device=dy.device)
    _lib.check(lib.semseg_bn_bwd_apply(_ptr(dy), _lo(dy), dp, _ptr(y), _lo(y), yp, _ptr(x), _lo(x), xp,
                                       _ptr(mean_invstd), _ptr(gamma), _ptr(scale_shift), _ptr(sums), float(count),
                                       n * h * w, c, int(bool(relu)), _ptr(dx), _lo(dx), c, _ptr(dres), _lo(dres), c,
                                       _ptr(dgb), _stream()), "semseg_bn_bwd_apply")
    return dx, dres, dgb


def bn_bwd_frozen(dy, y, raw, gamma, beta, running_mean, running_var, eps, relu, want_dres=False, want_sums=True):
    """Backward of BatchNorm normalised with its running statistics (+ residual) (+ ReLU), one pass.
    The ReLU mask comes from `y`, or from `raw` when `y` is None (forward without residual). Returns
    (d_raw, dres or None, sums [2][C] = (dbeta, dgamma) or None); with `raw` None, the dgamma row is zero."""
    lib = _lib.load()
    n, h, w, c, dp = _nhwc_meta(dy)
    yp = _nhwc_meta(y)[4] if y is not None else 0
    rp = _nhwc_meta(raw)[4] if raw is not None else 0
    _same_form(dy, y, raw)
    split = is_split(dy)
    m = n * h * w
    d_raw = empty_act((n, h, w, c), split, dy.device)
    dres = empty_act((n, h, w, c), split, dy.device) if want_dres else None
    ws, nf, sums = None, 0, None
    if want_sums:
        ws, nf = bn_workspace(m, c, dy.device)
        sums = torch.empty((2, c), dtype=torch.float32, device=dy.device)
    _lib.check(lib.semseg_bn_bwd_frozen(_ptr(dy), _lo(dy), dp, _ptr(y), _lo(y), yp, _ptr(raw), _lo(raw), rp,
                                        _ptr(gamma), _ptr(beta), _ptr(running_mean), _ptr(running_var), float(eps), m,
                                        c, int(bool(relu)), _ptr(d_raw), _lo(d_raw), c, _ptr(dres), _lo(dres), c,
                                        _ptr(ws), nf, _ptr(sums), _stream()), "semseg_bn_bwd_frozen")
    return d_raw, dres, sums


def add_act(a, b, out=None):
    """a + b of two activations (either storage form; a split-aware add, unlike adding the planes)."""
    lib = _lib.load()
    n, h, w, c, ap = _nhwc_meta(a)
    bp = _nhwc_meta(b)[4]
    if out is None:
        out = empty_act((n, h, w, c), is_split(a), a.device)
    op = _nhwc_meta(out)[4]
    _same_form(a, b, out)
    _lib.check(lib.semseg_add_act(_ptr(a), _lo(a), ap, _ptr(b), _lo(b), bp, _ptr(out), _lo(out), op, n * h * w, c,
                                  _stream()), "semseg_add_act")
    return out


def scale_nc(x, scale):
    """x[n, :, :, c] * scale[n, c] (scale fp32 [N, C]): Dropout2d's per-(image, channel) factor."""
    lib = _lib.load()
    n, h, w, c, xp = _nhwc_meta(x)
    assert scale.dtype == torch.float32 and scale.is_contiguous() and scale.numel() == n * c
    out = empty_act((n, h, w, c), is_split(x), x.device)
    _lib.check(lib.semseg_scale_nc(_ptr(x), _lo(x), xp, _ptr(scale), _ptr(out), _lo(out), c, n, h * w, c, _stream()),
               "semseg_scale_nc")
    return out


def fp_fork(x, scale):
    """Feature-perturbation fork of an N-image activation: the 2N-image cat(x, scale_nc(x, scale)) in x's storage form,
    from one read of x (scale fp32 [N, C])."""
    lib = _lib.load()
    n, h, w, c, xp = _nhwc_meta(x)
    assert scale.dtype == torch.float32 and scale.is_contiguous() and scale.numel() == n * c
    out = empty_act((2 * n, h, w, c), is_split(x), x.device)
    _lib.check(lib.semseg_fp_fork(_ptr(x), _lo(x), xp, _ptr(scale), _ptr(out), _lo(out), c, n, h * w, c, _stream()),
               "semseg_fp_fork")
    return out


def fp_fold(d, scale):
    """The fork's backward: d[:N] + scale * d[N:] of a 2N-image activation gradient, in fp32, rounded once."""
    lib = _lib.load()
    n2, h, w, c, dp = _nhwc_meta(d)
    assert n2 % 2 == 0, "the fold takes a 2N-image gradient"
    n = n2 // 2
    assert scale.dtype == torch.float32 and scale.is_contiguous() and scale.numel() == n * c
    out = empty_act((n, h, w, c), is_split(d), d.device)
    _lib.check(lib.semseg_fp_fold(_ptr(d), _lo(d), dp, _ptr(scale), _ptr(out), _lo(out), c, n, h * w, c, _stream()),
               "semseg_fp_fold")
    return out


def fp_fork_prefix(x, scale):
    """Feature-perturbation fork of an M-image activation whose first N images are perturbed (scale fp32 [N, C],
    N <= M): the (M + N)-image cat(x, scale_nc(x[:N], scale)) in x's storage form, from one read of x. M = N is fp_fork's
    result bit for bit."""
    lib = _lib.load()
    m, h, w, c, xp = _nhwc_meta(x)
    assert scale.dtype == torch.float32 and scale.is_contiguous() and scale.dim() == 2 and scale.shape[1] == c
    n = scale.shape[0]
    out = empty_act((m + n, h, w, c), is_split(x), x.device)
    _lib.check(lib.semseg_fp_fork_prefix(_ptr(x), _lo(x), xp, _ptr(scale), _ptr(out), _lo(out), c, m, n, h * w, c,
                                         _stream()),
               "semseg_fp_fork_prefix")
    return out


def fp_fold_prefix(d, scale):
    """fp_fork_prefix's backward: d[:M] with scale * d[M:] added to its first N images, of an (M + N)-image activation
    gradient (scale fp32 [N, C]), in fp32, rounded once. M = N is fp_fold's result bit for bit."""
    lib = _lib.load()
    mn, h, w, c, dp = _nhwc_meta(d)
    assert scale.dtype == torch.float32 and scale.is_contiguous() and scale.dim() == 2 and scale.shape[1] == c
    n = scale.shape[0]
    m = mn - n
    out = empty_act((m, h, w, c), is_split(d), d.device)
    _lib.check(lib.semseg_fp_fold_prefix(_ptr(d), _lo(d), dp, _ptr(scale), _ptr(out), _lo(out), c, m, n, h * w, c,
                                         _stream()),
               "semseg_fp_fold_prefix")
    return out


def f32_to_act(x, split, pad_to=8):
    """fp32 NHWC [N,H,W,C] (channel-contiguous, any pixel pitch) -> activation [N,H,W,Cp], Cp = C rounded up to
    `pad_to`, padding zero filled."""
    _require_cuda(x)
    lib = _lib.load()
    assert x.dtype == torch.float32 and x.dim() == 4 and x.stride(-1) == 1
    n, h, w, c = x.shape
    sn, sh, sw, _ = x.stride()
    assert sh == sw * w and sn == sh * h
    cp = round_up(c, pad_to)
    out = empty_act((n, h, w, cp), split, x.device)
    _lib.check(lib.semseg_f32_to_act(_ptr(x), sw, _ptr(out), _lo(out), cp, n * h * w, c, cp, _stream()),
               "semseg_f32_to_act")
    return out


def act_to_f32(x):
    """activation -> fp32 NHWC [N,H,W,C]."""
    lib = _lib.load()
    n, h, w, c, p = _nhwc_meta(x)
    out = torch.empty((n, h, w, c), dtype=torch.float32, device=x.device)
    _lib.check(lib.semseg_act_to_f32(_ptr(x), _lo(x), p, _ptr(out), c, n * h * w, c, _stream()), "semseg_act_to_f32")
    return out


# ------------------------------------------------------------------------------------------------ fused tail
def upsample_ce_fwd(logits, target, ignore_index, want_argmax=True, zoom=8):
    """logits fp32 NHWC [N,h,w,C], target int64 [N,Ho,Wo] with Ho = zoom*(h-1)+1, Wo = zoom*(w-1)+1 (zoom 1, 2, 4 or 8)
    -> (loss_info [2] = (mean CE, count), argmax, lse)."""
    _require_cuda(logits, target)
    lib = _lib.load()
    assert logits.dtype == torch.float32 and logits.dim() == 4 and logits.stride(-1) == 1
    assert target.dtype == torch.int64 and target.is_contiguous()
    n, h, w, c = logits.shape
    _, ho, wo = target.shape
    nws = int(lib.semseg_upsample_ce_zoom_workspace_floats(n, ho, wo, int(zoom)))
    _lib.check(0 if nws >= 0 else nws, "semseg_upsample_ce_zoom_workspace_floats")
    ws = torch.empty((nws,), dtype=torch.float32, device=logits.device)
    info = torch.empty((2,), dtype=torch.float32, device=logits.device)
    amax = torch.empty((n, ho, wo), dtype=torch.int64, device=logits.device) if want_argmax else None
    lse = torch.empty((n, ho, wo), dtype=torch.float32, device=logits.device)
    _lib.check(lib.semseg_upsample_ce_zoom_fwd(_ptr(logits), logits.stride(2), n, h, w, c, _ptr(target), ho, wo,
                                               int(zoom), int(ignore_index), _ptr(ws), _ptr(info), _ptr(amax),
                                               _ptr(lse), _stream()),
               "semseg_upsample_ce_zoom_fwd")
    return info, amax, lse


def upsample_ce_bwd(logits, target, ignore_index, lse, info, grad_out, zoom=8):
    lib = _lib.load()
    n, h, w, c = logits.shape
    _, ho, wo = target.shape
    dl = torch.empty((n, h, w, c), dtype=torch.float32, device=logits.device)
    nws = int(lib.semseg_upsample_ce_zoom_bwd_workspace_floats(n, ho, w, c, int(zoom)))
    _lib.check(0 if nws >= 0 else nws, "semseg_upsample_ce_zoom_bwd_workspace_floats")
    ws = torch.empty((nws,), dtype=torch.float32, device=logits.device)
    g = grad_out.reshape(1).float().contiguous()
    _lib.check(lib.semseg_upsample_ce_zoom_bwd(_ptr(logits), logits.stride(2), n, h, w, c, _ptr(target), ho, wo,
                                               int(zoom), int(ignore_index), _ptr(lse), _ptr(info), _ptr(g), _ptr(ws),
                                               _ptr(dl), _stream()),
               "semseg_upsample_ce_zoom_bwd")
    return dl


def _check_class_weight(weight, logits):
    """A class-weight tensor the weighted tail kernels read: None, or fp32 contiguous [C] on the logits' device."""
    if weight is None:
        return
    c = logits.shape[-1]
    if not (weight.dtype == torch.float32 and weight.dim() == 1 and weight.is_contiguous() and weight.numel() == c
            and weight.device == logits.device):
        raise ValueError("semseg_b200: class weights must be a contiguous fp32 [%d] tensor on %s, got %s %s on %s" %
                         (c, logits.device, weight.dtype, tuple(weight.shape), weight.device))


def upsample_ce_weighted_fwd(logits, target, ignore_index, weight, label_smoothing, want_argmax=True, zoom=8):
    """Class-weighted, label-smoothed cross-entropy on the fused tail (include/semseg_b200.h states the contract):
    arguments as upsample_ce_fwd plus `weight` (fp32 [C] or None = all ones) and `label_smoothing` in [0, 1]
    -> (loss_info [2] = (loss, D = sum of the valid pixels' target weights), argmax, lse)."""
    _require_cuda(logits, target)
    lib = _lib.load()
    assert logits.dtype == torch.float32 and logits.dim() == 4 and logits.stride(-1) == 1
    assert target.dtype == torch.int64 and target.is_contiguous()
    _check_class_weight(weight, logits)
    n, h, w, c = logits.shape
    _, ho, wo = target.shape
    nws = int(lib.semseg_upsample_ce_weighted_workspace_floats(n, ho, wo, int(zoom)))
    _lib.check(0 if nws >= 0 else nws, "semseg_upsample_ce_weighted_workspace_floats")
    ws = torch.empty((nws,), dtype=torch.float32, device=logits.device)
    info = torch.empty((2,), dtype=torch.float32, device=logits.device)
    amax = torch.empty((n, ho, wo), dtype=torch.int64, device=logits.device) if want_argmax else None
    lse = torch.empty((n, ho, wo), dtype=torch.float32, device=logits.device)
    _lib.check(lib.semseg_upsample_ce_weighted_fwd(_ptr(logits), logits.stride(2), n, h, w, c, _ptr(target), ho, wo,
                                                   int(zoom), int(ignore_index), _ptr(weight), float(label_smoothing),
                                                   _ptr(ws), _ptr(info), _ptr(amax), _ptr(lse), _stream()),
               "semseg_upsample_ce_weighted_fwd")
    return info, amax, lse


def upsample_ce_weighted_bwd(logits, target, ignore_index, weight, label_smoothing, lse, info, grad_out, zoom=8):
    lib = _lib.load()
    _check_class_weight(weight, logits)
    n, h, w, c = logits.shape
    _, ho, wo = target.shape
    dl = torch.empty((n, h, w, c), dtype=torch.float32, device=logits.device)
    nws = int(lib.semseg_upsample_ce_weighted_bwd_workspace_floats(n, ho, w, c, int(zoom)))
    _lib.check(0 if nws >= 0 else nws, "semseg_upsample_ce_weighted_bwd_workspace_floats")
    ws = torch.empty((nws,), dtype=torch.float32, device=logits.device)
    g = grad_out.reshape(1).float().contiguous()
    _lib.check(lib.semseg_upsample_ce_weighted_bwd(_ptr(logits), logits.stride(2), n, h, w, c, _ptr(target), ho, wo,
                                                   int(zoom), int(ignore_index), _ptr(weight), float(label_smoothing),
                                                   _ptr(lse), _ptr(info), _ptr(g), _ptr(ws), _ptr(dl), _stream()),
               "semseg_upsample_ce_weighted_bwd")
    return dl


def upsample_ce_ohem_fwd(logits, target, ignore_index, thresh, min_kept, want_argmax=True, zoom=8, weight=None):
    """OHEM cross-entropy on the fused tail (semseg_b200/losses.py states the contract); arguments as upsample_ce_fwd
    -> (loss_info [2] = (mean nll over the kept pixels, kept count), argmax, lse, p_t, nll, thr [1]). p_t / nll fp32
    [N,Ho,Wo], p_t = -1 where the pixel is not valid. `weight` (fp32 [C]): the weighted form, nll = w_t * nll."""
    _require_cuda(logits, target)
    lib = _lib.load()
    assert logits.dtype == torch.float32 and logits.dim() == 4 and logits.stride(-1) == 1
    assert target.dtype == torch.int64 and target.is_contiguous()
    _check_class_weight(weight, logits)
    n, h, w, c = logits.shape
    _, ho, wo = target.shape
    nws = int(lib.semseg_upsample_ce_ohem_workspace_floats(n, ho, wo, int(zoom)))
    _lib.check(0 if nws >= 0 else nws, "semseg_upsample_ce_ohem_workspace_floats")
    dev = logits.device
    ws = torch.empty((nws,), dtype=torch.float32, device=dev)
    info = torch.empty((2,), dtype=torch.float32, device=dev)
    thr = torch.empty((1,), dtype=torch.float32, device=dev)
    amax = torch.empty((n, ho, wo), dtype=torch.int64, device=dev) if want_argmax else None
    lse, pt, nll = (torch.empty((n, ho, wo), dtype=torch.float32, device=dev) for _ in range(3))
    head = (_ptr(logits), logits.stride(2), n, h, w, c, _ptr(target), ho, wo, int(zoom), int(ignore_index),
            float(thresh), int(min_kept))
    outs = (_ptr(ws), _ptr(info), _ptr(amax), _ptr(lse), _ptr(pt), _ptr(nll), _ptr(thr), _stream())
    if weight is None:
        _lib.check(lib.semseg_upsample_ce_ohem_fwd(*head, *outs), "semseg_upsample_ce_ohem_fwd")
    else:
        _lib.check(lib.semseg_upsample_ce_ohem_weighted_fwd(*head, _ptr(weight), *outs),
                   "semseg_upsample_ce_ohem_weighted_fwd")
    return info, amax, lse, pt, nll, thr


def upsample_ce_ohem_bwd(logits, target, ignore_index, lse, pt, thr, info, grad_out, zoom=8, weight=None):
    lib = _lib.load()
    _check_class_weight(weight, logits)
    n, h, w, c = logits.shape
    _, ho, wo = target.shape
    dl = torch.empty((n, h, w, c), dtype=torch.float32, device=logits.device)
    nws = int(lib.semseg_upsample_ce_ohem_bwd_workspace_floats(n, ho, w, c, int(zoom)))
    _lib.check(0 if nws >= 0 else nws, "semseg_upsample_ce_ohem_bwd_workspace_floats")
    ws = torch.empty((nws,), dtype=torch.float32, device=logits.device)
    g = grad_out.reshape(1).float().contiguous()
    head = (_ptr(logits), logits.stride(2), n, h, w, c, _ptr(target), ho, wo, int(zoom), int(ignore_index))
    tail = (_ptr(lse), _ptr(pt), _ptr(thr), _ptr(info), _ptr(g), _ptr(ws), _ptr(dl), _stream())
    if weight is None:
        _lib.check(lib.semseg_upsample_ce_ohem_bwd(*head, *tail), "semseg_upsample_ce_ohem_bwd")
    else:
        _lib.check(lib.semseg_upsample_ce_ohem_weighted_bwd(*head, _ptr(weight), *tail),
                   "semseg_upsample_ce_ohem_weighted_bwd")
    return dl


def upsample_ce_dice_fwd(logits, target, ignore_index, smooth, eps, ce_weight, want_argmax=True, zoom=8):
    """Soft Dice loss (+ ce_weight * CE) on the fused tail (include/semseg_b200.h states the contract); arguments as
    upsample_ce_fwd plus the Dice options -> (loss_info [2] = (loss, valid count), argmax, lse, table [5C+2] =
    (alpha, beta, I, S, n per class, ce_weight / n_valid, 1))."""
    _require_cuda(logits, target)
    lib = _lib.load()
    assert logits.dtype == torch.float32 and logits.dim() == 4 and logits.stride(-1) == 1
    assert target.dtype == torch.int64 and target.is_contiguous()
    n, h, w, c = logits.shape
    _, ho, wo = target.shape
    nws = int(lib.semseg_upsample_ce_dice_workspace_floats(n, ho, wo, c, int(zoom)))
    _lib.check(0 if nws >= 0 else nws, "semseg_upsample_ce_dice_workspace_floats")
    dev = logits.device
    ws = torch.empty((nws,), dtype=torch.float32, device=dev)
    info = torch.empty((2,), dtype=torch.float32, device=dev)
    table = torch.empty((5 * c + 2,), dtype=torch.float32, device=dev)
    amax = torch.empty((n, ho, wo), dtype=torch.int64, device=dev) if want_argmax else None
    lse = torch.empty((n, ho, wo), dtype=torch.float32, device=dev)
    _lib.check(lib.semseg_upsample_ce_dice_fwd(_ptr(logits), logits.stride(2), n, h, w, c, _ptr(target), ho, wo,
                                               int(zoom), int(ignore_index), float(smooth), float(eps),
                                               float(ce_weight), _ptr(ws), _ptr(info), _ptr(amax), _ptr(lse),
                                               _ptr(table), _stream()),
               "semseg_upsample_ce_dice_fwd")
    return info, amax, lse, table


def upsample_ce_dice_bwd(logits, target, ignore_index, lse, table, grad_out, zoom=8):
    lib = _lib.load()
    n, h, w, c = logits.shape
    _, ho, wo = target.shape
    dl = torch.empty((n, h, w, c), dtype=torch.float32, device=logits.device)
    nws = int(lib.semseg_upsample_ce_dice_bwd_workspace_floats(n, ho, wo, w, c, int(zoom)))
    _lib.check(0 if nws >= 0 else nws, "semseg_upsample_ce_dice_bwd_workspace_floats")
    ws = torch.empty((nws,), dtype=torch.float32, device=logits.device)
    g = grad_out.reshape(1).float().contiguous()
    _lib.check(lib.semseg_upsample_ce_dice_bwd(_ptr(logits), logits.stride(2), n, h, w, c, _ptr(target), ho, wo,
                                               int(zoom), int(ignore_index), _ptr(lse), _ptr(table), _ptr(g), _ptr(ws),
                                               _ptr(dl), _stream()),
               "semseg_upsample_ce_dice_bwd")
    return dl


def upsample_ce_focal_fwd(logits, target, ignore_index, weight, gamma, want_argmax=True, zoom=8):
    """Softmax focal loss on the fused tail (include/semseg_b200.h states the contract); arguments as upsample_ce_fwd
    plus `weight` (fp32 [C] or None = all ones) and `gamma` >= 0 -> (loss_info [2] = (loss, valid count), argmax, lse,
    mod). mod fp32 [N,Ho,Wo]: each pixel's gradient modulator w_t * M, 0 where the pixel is not valid."""
    _require_cuda(logits, target)
    lib = _lib.load()
    assert logits.dtype == torch.float32 and logits.dim() == 4 and logits.stride(-1) == 1
    assert target.dtype == torch.int64 and target.is_contiguous()
    _check_class_weight(weight, logits)
    n, h, w, c = logits.shape
    _, ho, wo = target.shape
    nws = int(lib.semseg_upsample_ce_focal_workspace_floats(n, ho, wo, int(zoom)))
    _lib.check(0 if nws >= 0 else nws, "semseg_upsample_ce_focal_workspace_floats")
    dev = logits.device
    ws = torch.empty((nws,), dtype=torch.float32, device=dev)
    info = torch.empty((2,), dtype=torch.float32, device=dev)
    amax = torch.empty((n, ho, wo), dtype=torch.int64, device=dev) if want_argmax else None
    lse, mod = (torch.empty((n, ho, wo), dtype=torch.float32, device=dev) for _ in range(2))
    _lib.check(lib.semseg_upsample_ce_focal_fwd(_ptr(logits), logits.stride(2), n, h, w, c, _ptr(target), ho, wo,
                                                int(zoom), int(ignore_index), _ptr(weight), float(gamma), _ptr(ws),
                                                _ptr(info), _ptr(amax), _ptr(lse), _ptr(mod), _stream()),
               "semseg_upsample_ce_focal_fwd")
    return info, amax, lse, mod


def upsample_ce_focal_bwd(logits, target, ignore_index, lse, mod, info, grad_out, zoom=8):
    lib = _lib.load()
    n, h, w, c = logits.shape
    _, ho, wo = target.shape
    dl = torch.empty((n, h, w, c), dtype=torch.float32, device=logits.device)
    nws = int(lib.semseg_upsample_ce_focal_bwd_workspace_floats(n, ho, w, c, int(zoom)))
    _lib.check(0 if nws >= 0 else nws, "semseg_upsample_ce_focal_bwd_workspace_floats")
    ws = torch.empty((nws,), dtype=torch.float32, device=logits.device)
    g = grad_out.reshape(1).float().contiguous()
    _lib.check(lib.semseg_upsample_ce_focal_bwd(_ptr(logits), logits.stride(2), n, h, w, c, _ptr(target), ho, wo,
                                                int(zoom), int(ignore_index), _ptr(lse), _ptr(mod), _ptr(info), _ptr(g),
                                                _ptr(ws), _ptr(dl), _stream()),
               "semseg_upsample_ce_focal_bwd")
    return dl


def upsample_ce_lovasz_fwd(logits, target, ignore_index, classes_all, per_image, ce_weight, want_argmax=True, zoom=8,
                           return_workspace=False):
    """Lovász-Softmax loss (+ ce_weight * CE) on the fused tail (include/semseg_b200.h states the contract) ->
    (loss_info [2] = (loss, valid count), argmax, lse, gamma [N*H*W*C + 2]); with return_workspace also the forward
    workspace, whose first 2 S L words are the sorted keys and payloads of every considered segment."""
    _require_cuda(logits, target)
    lib = _lib.load()
    assert logits.dtype == torch.float32 and logits.dim() == 4 and logits.stride(-1) == 1
    assert target.dtype == torch.int64 and target.is_contiguous()
    n, h, w, c = logits.shape
    _, ho, wo = target.shape
    nws = int(lib.semseg_upsample_ce_lovasz_workspace_floats(n, ho, wo, c, int(zoom), int(bool(per_image))))
    _lib.check(0 if nws >= 0 else nws, "semseg_upsample_ce_lovasz_workspace_floats")
    dev = logits.device
    ws = torch.empty((nws,), dtype=torch.float32, device=dev)
    info = torch.empty((2,), dtype=torch.float32, device=dev)
    gamma = torch.empty((n * ho * wo * c + 2,), dtype=torch.float32, device=dev)
    amax = torch.empty((n, ho, wo), dtype=torch.int64, device=dev) if want_argmax else None
    lse = torch.empty((n, ho, wo), dtype=torch.float32, device=dev)
    _lib.check(lib.semseg_upsample_ce_lovasz_fwd(_ptr(logits), logits.stride(2), n, h, w, c, _ptr(target), ho, wo,
                                                 int(zoom), int(ignore_index), int(bool(classes_all)),
                                                 int(bool(per_image)), float(ce_weight), _ptr(ws), _ptr(info),
                                                 _ptr(amax), _ptr(lse), _ptr(gamma), _stream()),
               "semseg_upsample_ce_lovasz_fwd")
    if return_workspace:
        return info, amax, lse, gamma, ws
    return info, amax, lse, gamma


def upsample_ce_lovasz_bwd(logits, target, ignore_index, lse, gamma, grad_out, zoom=8):
    lib = _lib.load()
    n, h, w, c = logits.shape
    _, ho, wo = target.shape
    dl = torch.empty((n, h, w, c), dtype=torch.float32, device=logits.device)
    nws = int(lib.semseg_upsample_ce_lovasz_bwd_workspace_floats(n, ho, wo, w, c, int(zoom)))
    _lib.check(0 if nws >= 0 else nws, "semseg_upsample_ce_lovasz_bwd_workspace_floats")
    ws = torch.empty((nws,), dtype=torch.float32, device=logits.device)
    g = grad_out.reshape(1).float().contiguous()
    _lib.check(lib.semseg_upsample_ce_lovasz_bwd(_ptr(logits), logits.stride(2), n, h, w, c, _ptr(target), ho, wo,
                                                 int(zoom), int(ignore_index), _ptr(lse), _ptr(gamma), _ptr(g),
                                                 _ptr(ws), _ptr(dl), _stream()),
               "semseg_upsample_ce_lovasz_bwd")
    return dl


def _kd_map_meta(x):
    """(N, h, w, C, pitch) of an fp32 NHWC logit map whose pixels may be padded (a channel slice of a wider buffer)."""
    assert x.dtype == torch.float32 and x.dim() == 4 and x.stride(-1) == 1
    n, h, w, c = x.shape
    pitch = x.stride(2)
    assert x.stride(1) == w * pitch and x.stride(0) == h * x.stride(1), "logits must be pixel-contiguous"
    return n, h, w, c, pitch


def upsample_kd_fwd(student, teacher, temperature, zoom=8):
    """Pixel-wise distillation term on the fused tail (include/semseg_b200.h states the contract): student / teacher
    fp32 NHWC [N,h,w,C] maps (each with its own pixel pitch), both upsampled xzoom -> (kl_info [2] = (KL, P),
    lse [N,Ho,Wo,2] = (lse(s/T), lse(t/T)) per pixel)."""
    _require_cuda(student, teacher)
    lib = _lib.load()
    n, h, w, c, ps = _kd_map_meta(student)
    shape_t = _kd_map_meta(teacher)
    assert shape_t[:4] == (n, h, w, c), "student and teacher maps differ in shape"
    ho, wo = int(zoom) * (h - 1) + 1, int(zoom) * (w - 1) + 1
    nws = int(lib.semseg_upsample_kd_workspace_floats(n, ho, wo, int(zoom)))
    _lib.check(0 if nws >= 0 else nws, "semseg_upsample_kd_workspace_floats")
    dev = student.device
    ws = torch.empty((nws,), dtype=torch.float32, device=dev)
    info = torch.empty((2,), dtype=torch.float32, device=dev)
    lse = torch.empty((n, ho, wo, 2), dtype=torch.float32, device=dev)
    _lib.check(lib.semseg_upsample_kd_fwd(_ptr(student), ps, _ptr(teacher), shape_t[4], n, h, w, c, ho, wo, int(zoom),
                                          float(temperature), _ptr(ws), _ptr(info), _ptr(lse), _stream()),
               "semseg_upsample_kd_fwd")
    return info, lse


def upsample_kd_bwd(student, teacher, temperature, kd_weight, lse, grad_out, dlogits, zoom=8):
    """dlogits (fp32 [N,h,w,C], dense, already holding a gradient) += grad_out * d(kd_weight T^2 KL)/d student, in
    place; returns dlogits."""
    lib = _lib.load()
    n, h, w, c, ps = _kd_map_meta(student)
    pt = _kd_map_meta(teacher)[4]
    assert dlogits.shape == (n, h, w, c) and dlogits.dtype == torch.float32 and dlogits.is_contiguous()
    ho, wo = int(zoom) * (h - 1) + 1, int(zoom) * (w - 1) + 1
    nws = int(lib.semseg_upsample_kd_bwd_workspace_floats(n, ho, w, c, int(zoom)))
    _lib.check(0 if nws >= 0 else nws, "semseg_upsample_kd_bwd_workspace_floats")
    ws = torch.empty((nws,), dtype=torch.float32, device=student.device)
    g = grad_out.reshape(1).float().contiguous()
    _lib.check(lib.semseg_upsample_kd_bwd(_ptr(student), ps, _ptr(teacher), pt, n, h, w, c, ho, wo, int(zoom),
                                          float(temperature), float(kd_weight), _ptr(lse), _ptr(g), _ptr(ws),
                                          _ptr(dlogits), _stream()),
               "semseg_upsample_kd_bwd")
    return dlogits


def upsample_pl_fwd(student, teacher, target, ignore_index, threshold, pl_weight, ce_weight, want_argmax=True,
                    zoom=8, mix_mask=None):
    """Confidence-masked pseudo-label cross-entropy on the fused tail (include/semseg_b200.h states the contract):
    student / teacher fp32 NHWC [N,h,w,C] maps (each with its own pixel pitch), target int64 [N,Ho,Wo] ->
    (loss_info [6] = (CE mean over L, |L|, PL sum / |U|, |U|, 0, 1), argmax, lse, effective target int64 [N,Ho,Wo],
    weight fp32 [N,Ho,Wo]). The backward is upsample_ce_focal_bwd(student, eff, -1, lse, weight, loss_info[4:], ...).
    mix_mask (uint8 [N, 8(h-1)+1, 8(w-1)+1], mix_apply's mask): the mixed form, each pixel's teacher image n or
    (n + 1) mod N as the mask says (semseg_upsample_pl_mix_fwd)."""
    _require_cuda(student, teacher, target, mix_mask)
    lib = _lib.load()
    n, h, w, c, ps = _kd_map_meta(student)
    shape_t = _kd_map_meta(teacher)
    assert shape_t[:4] == (n, h, w, c), "student and teacher maps differ in shape"
    assert target.dtype == torch.int64 and target.is_contiguous()
    _, ho, wo = target.shape
    nws = int(lib.semseg_upsample_pl_workspace_floats(n, ho, wo, int(zoom)))
    _lib.check(0 if nws >= 0 else nws, "semseg_upsample_pl_workspace_floats")
    dev = student.device
    ws = torch.empty((nws,), dtype=torch.float32, device=dev)
    info = torch.empty((6,), dtype=torch.float32, device=dev)
    amax = torch.empty((n, ho, wo), dtype=torch.int64, device=dev) if want_argmax else None
    eff = torch.empty((n, ho, wo), dtype=torch.int64, device=dev)
    lse, wt = (torch.empty((n, ho, wo), dtype=torch.float32, device=dev) for _ in range(2))
    if mix_mask is None:
        _lib.check(lib.semseg_upsample_pl_fwd(_ptr(student), ps, _ptr(teacher), shape_t[4], n, h, w, c, _ptr(target),
                                              ho, wo, int(zoom), int(ignore_index), float(threshold), float(pl_weight),
                                              float(ce_weight), _ptr(ws), _ptr(info), _ptr(amax), _ptr(lse), _ptr(eff),
                                              _ptr(wt), _stream()),
                   "semseg_upsample_pl_fwd")
    else:
        assert mix_mask.dtype == torch.uint8 and mix_mask.is_contiguous()
        assert tuple(mix_mask.shape) == (n, 8 * (h - 1) + 1, 8 * (w - 1) + 1), "mix mask is not on the input grid"
        _lib.check(lib.semseg_upsample_pl_mix_fwd(_ptr(student), ps, _ptr(teacher), shape_t[4], n, h, w, c,
                                                  _ptr(target), ho, wo, int(zoom), int(ignore_index), float(threshold),
                                                  float(pl_weight), float(ce_weight), _ptr(mix_mask), _ptr(ws),
                                                  _ptr(info), _ptr(amax), _ptr(lse), _ptr(eff), _ptr(wt), _stream()),
                   "semseg_upsample_pl_mix_fwd")
    return info, amax, lse, eff, wt


MIX_MODES = {'cutmix': 0, 'classmix': 1}      # SEMSEG_MIX_CUTMIX, SEMSEG_MIX_CLASSMIX


def mix_argmax_x8(teacher):
    """The teacher's argmax after the x8 bilinear (align_corners) upsample (include/semseg_b200.h
    semseg_mix_argmax_x8): fp32 NHWC [N,h,w,C] (padded pitch allowed) -> (argmax uint8 [N, 8(h-1)+1, 8(w-1)+1],
    present int32 [N, 8]: the classes that occur in each image, as 256 bits)."""
    _require_cuda(teacher)
    lib = _lib.load()
    n, h, w, c, pitch = _kd_map_meta(teacher)
    amap = torch.empty((n, 8 * (h - 1) + 1, 8 * (w - 1) + 1), dtype=torch.uint8, device=teacher.device)
    present = torch.empty((n, 8), dtype=torch.int32, device=teacher.device)
    _lib.check(lib.semseg_mix_argmax_x8(_ptr(teacher), pitch, n, h, w, c, _ptr(amap), _ptr(present), _stream()),
               "semseg_mix_argmax_x8")
    return amap, present


def mix_select(uniforms, present, classes):
    """ClassMix's class sets (semseg_mix_select): uniforms fp32 [N, >= 5 + classes], present int32 [N, 8] -> selected
    int32 [N, 8], the ceil(k/2) present classes of each image with the smallest (u[n, 5 + c], c), as bits."""
    _require_cuda(uniforms, present)
    lib = _lib.load()
    assert uniforms.dtype == torch.float32 and uniforms.dim() == 2 and uniforms.stride(1) == 1
    assert present.dtype == torch.int32 and present.is_contiguous() and present.shape == (uniforms.shape[0], 8)
    sel = torch.empty_like(present)
    _lib.check(lib.semseg_mix_select(_ptr(uniforms), uniforms.stride(0), _ptr(present), uniforms.shape[0],
                                     int(classes), _ptr(sel), _stream()),
               "semseg_mix_select")
    return sel


def mix_apply(mode, x, y, uniforms, p, area, ratio, zoom, amap=None, selected=None):
    """The mixed batch (semseg_mix_apply): x fp32 NCHW [N,Cin,H,W], y int64 [N,Ho,Wo], uniforms fp32 [N, >= 5] ->
    (mask uint8 [N,H,W], x_mixed, y_mixed). mode 'cutmix' or 'classmix' (the latter with mix_argmax_x8's argmax and
    mix_select's selection); p, area = (lo, hi), ratio = (lo, hi) as losses.MixPseudoLabelLoss takes them."""
    _require_cuda(x, y, uniforms, amap, selected)
    lib = _lib.load()
    assert x.dtype == torch.float32 and x.dim() == 4 and x.is_contiguous()
    assert y.dtype == torch.int64 and y.dim() == 3 and y.is_contiguous()
    assert uniforms.dtype == torch.float32 and uniforms.dim() == 2 and uniforms.stride(1) == 1
    n, cin, hh, ww = x.shape
    assert y.shape[0] == n and uniforms.shape[0] == n, "input, target and uniforms differ in batch size"
    if mode == 'classmix':
        assert amap is not None and amap.dtype == torch.uint8 and amap.is_contiguous() and amap.shape == (n, hh, ww)
        assert selected is not None and selected.dtype == torch.int32 and selected.is_contiguous() and \
            selected.shape == (n, 8)
    mask = torch.empty((n, hh, ww), dtype=torch.uint8, device=x.device)
    xm = torch.empty_like(x)
    ym = torch.empty_like(y)
    _lib.check(lib.semseg_mix_apply(MIX_MODES[mode], _ptr(x), n, cin, hh, ww, _ptr(y), y.shape[1], y.shape[2],
                                    int(zoom), _ptr(uniforms), uniforms.stride(0), float(p), float(area[0]),
                                    float(area[1]), float(ratio[0]), float(ratio[1]), _ptr(amap), _ptr(selected),
                                    _ptr(mask), _ptr(xm), _ptr(ym), _stream()),
               "semseg_mix_apply")
    return mask, xm, ym


def ema_multi(items_dev, n_items, n_chunks, decay):
    """shadow <- lerp(shadow, source, 1 - decay) for every fp32 item, int64 items copied, in one launch
    (include/semseg_b200.h semseg_ema_multi); `items_dev` is a device uint8 tensor holding the item table."""
    lib = _lib.load()
    _lib.check(lib.semseg_ema_multi(_ptr(items_dev), int(n_items), int(n_chunks), float(decay), _stream()),
               "semseg_ema_multi")


def segsort_u32_pairs(keys, vals, skip=None):
    """Stable sort of each row of the int32 [S, L] CUDA tensors `keys` / `vals` (uint32 bit patterns) by key, in place;
    rows whose int32 `skip` [S] entry is non-zero are left untouched."""
    _require_cuda(keys, vals)
    lib = _lib.load()
    assert keys.dtype == vals.dtype == torch.int32 and keys.shape == vals.shape and keys.dim() == 2
    assert keys.is_contiguous() and vals.is_contiguous()
    s, l = keys.shape
    nb = int(lib.semseg_segsort_u32_pairs_workspace_bytes(s, l))
    _lib.check(0 if nb >= 0 else nb, "semseg_segsort_u32_pairs_workspace_bytes")
    ws = torch.empty((nb,), dtype=torch.uint8, device=keys.device)
    ka, va = torch.empty_like(keys), torch.empty_like(vals)
    if skip is not None:
        assert skip.dtype == torch.int32 and skip.is_contiguous() and skip.numel() == s
    _lib.check(lib.semseg_segsort_u32_pairs(_ptr(keys), _ptr(vals), _ptr(ka), _ptr(va), s, l, _ptr(skip), _ptr(ws),
                                            _stream()),
               "semseg_segsort_u32_pairs")
    return keys, vals


def upsample_ce_rmi_fwd(logits, target, ignore_index, bce_weight, pos_alpha, ce_weight, want_argmax=True, zoom=8,
                        workspace=None):
    """RMI loss (+ bce_weight * BCE + ce_weight * CE) on the fused tail (include/semseg_b200.h states the contract);
    arguments as upsample_ce_fwd plus the RMI options -> (loss_info [5] = (loss, valid count, BCE, RMI, CE), argmax,
    lse, pooled [2, N, C, Ho/4, Wo/4] = (Y, Q), table [N*C*184 + 4]: per (n, c) [G_ab' | 2 G_bb], the means and r,
    then the backward's scalars). `workspace` (fp32, at least semseg_upsample_ce_rmi_workspace_floats, 8-byte aligned)
    lets a caller read the raw fp64 moment sums the kernels leave at its start."""
    _require_cuda(logits, target)
    lib = _lib.load()
    assert logits.dtype == torch.float32 and logits.dim() == 4 and logits.stride(-1) == 1
    assert target.dtype == torch.int64 and target.is_contiguous()
    n, h, w, c = logits.shape
    _, ho, wo = target.shape
    nws = int(lib.semseg_upsample_ce_rmi_workspace_floats(n, ho, wo, c, int(zoom)))
    _lib.check(0 if nws >= 0 else nws, "semseg_upsample_ce_rmi_workspace_floats")
    ntab = int(lib.semseg_upsample_ce_rmi_table_floats(n, c))
    _lib.check(0 if ntab >= 0 else ntab, "semseg_upsample_ce_rmi_table_floats")
    dev = logits.device
    if workspace is None:
        workspace = torch.empty((nws,), dtype=torch.float32, device=dev)
    assert workspace.dtype == torch.float32 and workspace.numel() >= nws and workspace.is_contiguous()
    info = torch.empty((5,), dtype=torch.float32, device=dev)
    table = torch.empty((ntab,), dtype=torch.float32, device=dev)
    pooled = torch.empty((2, n, c, ho // 4, wo // 4), dtype=torch.float32, device=dev)
    amax = torch.empty((n, ho, wo), dtype=torch.int64, device=dev) if want_argmax else None
    lse = torch.empty((n, ho, wo), dtype=torch.float32, device=dev)
    _lib.check(lib.semseg_upsample_ce_rmi_fwd(_ptr(logits), logits.stride(2), n, h, w, c, _ptr(target), ho, wo,
                                              int(zoom), int(ignore_index), float(bce_weight), float(pos_alpha),
                                              float(ce_weight), _ptr(workspace), _ptr(info), _ptr(amax), _ptr(lse),
                                              _ptr(pooled), _ptr(table), _stream()),
               "semseg_upsample_ce_rmi_fwd")
    return info, amax, lse, pooled, table


def upsample_ce_rmi_bwd(logits, target, ignore_index, lse, pooled, table, grad_out, zoom=8):
    lib = _lib.load()
    n, h, w, c = logits.shape
    _, ho, wo = target.shape
    dl = torch.empty((n, h, w, c), dtype=torch.float32, device=logits.device)
    nws = int(lib.semseg_upsample_ce_rmi_bwd_workspace_floats(n, ho, wo, w, c, int(zoom)))
    _lib.check(0 if nws >= 0 else nws, "semseg_upsample_ce_rmi_bwd_workspace_floats")
    ws = torch.empty((nws,), dtype=torch.float32, device=logits.device)
    g = grad_out.reshape(1).float().contiguous()
    _lib.check(lib.semseg_upsample_ce_rmi_bwd(_ptr(logits), logits.stride(2), n, h, w, c, _ptr(target), ho, wo,
                                              int(zoom), int(ignore_index), _ptr(lse), _ptr(pooled), _ptr(table),
                                              _ptr(g), _ptr(ws), _ptr(dl), _stream()),
               "semseg_upsample_ce_rmi_bwd")
    return dl


# ------------------------------------------------------------------------------------------------ sliding-window evaluation
def window_scores(logits, flip, out):
    """fp32 NHWC logits [G (+G mirrored crops when flip), h, w, C] -> flip-averaged softmax scores written into `out`,
    a contiguous fp32 [G, C, 8(h-1)+1, 8(w-1)+1] tensor (typically a slice of a scale's score buffer)."""
    _require_cuda(logits, out)
    lib = _lib.load()
    assert logits.dtype == torch.float32 and logits.dim() == 4 and logits.stride(3) == 1
    n, h, w, c = logits.shape
    pitch = logits.stride(2)
    assert logits.stride(1) == w * pitch and logits.stride(0) == h * logits.stride(1), "logits must be pixel-contiguous"
    g = n // 2 if flip else n
    assert not flip or n % 2 == 0, "flip needs the crops followed by their mirrors"
    assert out.dtype == torch.float32 and out.is_contiguous() and out.dim() == 4 and tuple(out.shape[:2]) == (g, c)
    _lib.check(lib.semseg_window_scores(_ptr(logits), pitch, g, h, w, c, int(bool(flip)), _ptr(out), out.shape[2],
                                        out.shape[3], _stream()), "semseg_window_scores")
    return out


def _int_array(vals):
    return (ctypes.c_int * len(vals))(*[int(v) for v in vals])


def window_accumulate(scores, ys, xs, full_size, top, left, img_size):
    """Overlap-normalised fp64 canvas [C, img_h, img_w] of a scale: scores fp32 [len(ys)*len(xs), C, crop_h, crop_w] of
    the crop grid (row-major), crop origins ys / xs on the padded image of size full_size, un-padded window at
    (top, left) of size img_size."""
    _require_cuda(scores)
    lib = _lib.load()
    assert scores.dtype == torch.float32 and scores.is_contiguous() and scores.dim() == 4
    k, c, ch, cw = scores.shape
    assert k == len(ys) * len(xs), "one score map per crop of the grid"
    img_h, img_w = img_size
    canvas = torch.empty((c, img_h, img_w), dtype=torch.float64, device=scores.device)
    _lib.check(lib.semseg_window_accumulate(_ptr(scores), c, ch, cw, _int_array(ys), len(ys), _int_array(xs), len(xs),
                                            full_size[0], full_size[1], top, left, img_h, img_w, _ptr(canvas),
                                            _stream()), "semseg_window_accumulate")
    return canvas


def window_resize_add(canvas, total):
    """total fp64 [C, H, W] += bilinear resize (align_corners=False) of canvas fp64 [C, h, w] to H x W; in place."""
    _require_cuda(canvas, total)
    lib = _lib.load()
    assert canvas.dtype == torch.float64 and total.dtype == torch.float64
    assert canvas.is_contiguous() and total.is_contiguous() and canvas.dim() == 3 and total.dim() == 3
    assert canvas.shape[0] == total.shape[0], "canvas and total must have the same classes"
    c, hi, wi = canvas.shape
    _, ho, wo = total.shape
    _lib.check(lib.semseg_window_resize_add(_ptr(canvas), c, hi, wi, _ptr(total), ho, wo, _stream()),
               "semseg_window_resize_add")
    return total


# ------------------------------------------------------------------------------------------------ pyramid pooling
def _bin_args(bins, tensors):
    """(bins[], hi pointers[], lo pointers[] or NULL, nb)"""
    nb = len(bins)
    barr = (ctypes.c_int * nb)(*bins)
    parr = (ctypes.c_void_p * nb)(*[t.data_ptr() for t in tensors])
    larr = (ctypes.c_void_p * nb)(*[_lo_int(t) for t in tensors]) if is_split(tensors[0]) else None
    return barr, parr, larr, nb


def ppm_pool(x, bins):
    """x NHWC bf16 -> [pooled_k [N,b,b,C] bf16 for b in bins] (AdaptiveAvgPool2d of every bin, one launch)."""
    _require_cuda(x)
    lib = _lib.load()
    n, h, w, c, p = _nhwc_meta(x)
    outs = [empty_act((n, b, b, c), is_split(x), x.device) for b in bins]
    barr, parr, larr, nb = _bin_args(bins, outs)
    _lib.check(lib.semseg_ppm_pool(_ptr(x), _lo(x), p, n, h, w, c, barr, parr, larr, nb, _stream()), "semseg_ppm_pool")
    return outs


def ppm_pool_bwd(dpooled, bins, n, h, w, c, add=None):
    """dx of ppm_pool; `add` (NHWC bf16, possibly a channel slice of a wider tensor) is summed in."""
    lib = _lib.load()
    dpooled = [d.contiguous() for d in dpooled]
    dx = empty_act((n, h, w, c), is_split(dpooled[0]), dpooled[0].device)
    barr, parr, larr, nb = _bin_args(bins, dpooled)
    ap = _nhwc_meta(add)[4] if add is not None else 0
    _same_form(dx, add)
    _lib.check(lib.semseg_ppm_pool_bwd(parr, larr, barr, nb, n, h, w, c, _ptr(dx), _lo(dx), c, _ptr(add), _lo(add), ap,
                                       _stream()), "semseg_ppm_pool_bwd")
    return dx


def ppm_upsample_concat(x, feats, bins):
    """-> out [N,H,W,C + nb*Cr] bf16 = cat([x, bilinear(feats_k)...], channel)."""
    lib = _lib.load()
    n, h, w, c, p = _nhwc_meta(x)
    feats = [f.contiguous() for f in feats]
    cr = feats[0].shape[-1]
    out = empty_act((n, h, w, c + len(bins) * cr), is_split(x), x.device)
    barr, parr, larr, nb = _bin_args(bins, feats)
    _same_form(x, feats[0])
    _lib.check(lib.semseg_ppm_upsample_concat(_ptr(x), _lo(x), p, parr, larr, barr, nb, n, h, w, c, cr, _ptr(out),
                                              _lo(out), out.shape[-1], _stream()), "semseg_ppm_upsample_concat")
    return out


def ppm_upsample_bwd(dout, c_off, bins, cr):
    lib = _lib.load()
    n, h, w, ct, p = _nhwc_meta(dout)
    dfeats = [empty_act((n, b, b, cr), is_split(dout), dout.device) for b in bins]
    barr, parr, larr, nb = _bin_args(bins, dfeats)
    _lib.check(lib.semseg_ppm_upsample_bwd(_ptr(dout), _lo(dout), p, c_off, parr, larr, barr, nb, n, h, w, cr,
                                           _stream()), "semseg_ppm_upsample_bwd")
    return dfeats


# ------------------------------------------------------------------------------------------------ bilinear resize
def resize_bilinear(x, size):
    """NHWC activation [N,Hi,Wi,C] -> [N,Ho,Wo,C], bilinear with align_corners=True."""
    _require_cuda(x)
    lib = _lib.load()
    n, hi, wi, c, p = _nhwc_meta(x)
    ho, wo = int(size[0]), int(size[1])
    y = empty_act((n, ho, wo, c), is_split(x), x.device)
    _lib.check(lib.semseg_resize_bilinear_fwd(_ptr(x), _lo(x), p, n, hi, wi, c, ho, wo, _ptr(y), _lo(y), c, _stream()),
               "semseg_resize_bilinear_fwd")
    return y


def resize_bilinear_bwd(dy, in_size):
    """Adjoint of resize_bilinear: dy [N,Ho,Wo,C] -> dx [N,Hi,Wi,C]."""
    lib = _lib.load()
    n, ho, wo, c, p = _nhwc_meta(dy)
    hi, wi = int(in_size[0]), int(in_size[1])
    dx = empty_act((n, hi, wi, c), is_split(dy), dy.device)
    _lib.check(lib.semseg_resize_bilinear_bwd(_ptr(dy), _lo(dy), p, n, hi, wi, c, ho, wo, _ptr(dx), _lo(dx), c, _stream()),
               "semseg_resize_bilinear_bwd")
    return dx


# ------------------------------------------------------------------------------------------------ max pool
def maxpool3x3s2_fwd(x, want_argcode=True):
    """-> (y, argcode uint8 or None)."""
    _require_cuda(x)
    lib = _lib.load()
    n, h, w, c, p = _nhwc_meta(x)
    assert p == c, "maxpool expects a dense NHWC tensor"
    shape = (n, (h - 1) // 2 + 1, (w - 1) // 2 + 1, c)
    y = empty_act(shape, is_split(x), x.device)
    code = torch.empty(shape, dtype=torch.uint8, device=x.device) if want_argcode else None
    _lib.check(lib.semseg_maxpool3x3s2_fwd(_ptr(x), _lo(x), _ptr(y), _lo(y), _ptr(code), n, h, w, c, _stream()),
               "semseg_maxpool3x3s2_fwd")
    return y, code


def maxpool3x3s2_bwd(argcode, dy, in_shape):
    lib = _lib.load()
    n, h, w, c = in_shape
    dy = dy.contiguous()
    dx = empty_act((n, h, w, c), is_split(dy), dy.device)
    _lib.check(lib.semseg_maxpool3x3s2_bwd(_ptr(argcode), _ptr(dy), _lo(dy), _ptr(dx), _lo(dx), n, h, w, c,
                                           _stream()), "semseg_maxpool3x3s2_bwd")
    return dx


# ------------------------------------------------------------------------------------------------ batch augmentation
def augment(data, descs, descs_dev, crop_h, crop_w, mean, std, ignore_label):
    """One semseg_augment launch. `data`: uint8 CUDA buffer of every sample's image and label; `descs`: ctypes array of
    AugmentDesc (validated on the host); `descs_dev`: the same bytes on the device. -> (fp32 [N,3,ch,cw], int64
    [N,ch,cw])."""
    _require_cuda(data, descs_dev)
    lib = _lib.load()
    assert data.dtype == torch.uint8 and data.is_contiguous()
    n = len(descs)
    img = torch.empty((n, 3, crop_h, crop_w), dtype=torch.float32, device=data.device)
    lab = torch.empty((n, crop_h, crop_w), dtype=torch.int64, device=data.device)
    m3, s3 = (ctypes.c_float * 3)(*mean), (ctypes.c_float * 3)(*std)
    _lib.check(lib.semseg_augment(_ptr(data), data.numel(), descs, _ptr(descs_dev), n, crop_h, crop_w, m3, s3,
                                  ignore_label, _ptr(img), _ptr(lab), _stream()), "semseg_augment")
    return img, lab


STRONG_TILE = 32          # csrc/strong.cu kStrongTile: one contrast partial per (32x32 tile, image)


def strong_augment(x, uniforms, brightness, contrast, saturation, hue, p_jitter, p_gray, p_blur, sigma, mean, std):
    """The strong view (semseg_strong_augment): x fp32 NCHW [N,3,H,W] (normalised), uniforms fp32 [N, >= 12] -> the
    view, a new tensor of x's shape. sigma = (lo, hi); mean / std: 3 numbers each, the normalisation of x."""
    _require_cuda(x, uniforms)
    lib = _lib.load()
    assert x.dtype == torch.float32 and x.dim() == 4 and x.is_contiguous()
    assert uniforms.dtype == torch.float32 and uniforms.dim() == 2 and uniforms.stride(1) == 1
    n, c, hh, ww = x.shape
    assert uniforms.shape[0] == n, "input and uniforms differ in batch size"
    out = torch.empty_like(x)
    ws = torch.empty((n * -(-hh // STRONG_TILE) * -(-ww // STRONG_TILE),), dtype=torch.float32, device=x.device)
    m3, s3 = (ctypes.c_float * 3)(*mean), (ctypes.c_float * 3)(*std)
    _lib.check(lib.semseg_strong_augment(_ptr(x), n, c, hh, ww, _ptr(uniforms), uniforms.stride(0), float(brightness),
                                         float(contrast), float(saturation), float(hue), float(p_jitter),
                                         float(p_gray), float(p_blur), float(sigma[0]), float(sigma[1]), m3, s3,
                                         _ptr(ws), _ptr(out), _stream()),
               "semseg_strong_augment")
    return out
