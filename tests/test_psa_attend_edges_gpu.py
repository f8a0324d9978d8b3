"""GPU tier (-m gpu): the fused point-wise spatial attention kernels (csrc/psa_fused.cu: psa_attend_kernel in its forward
and feature-gradient instances, psa_attn_grad_kernel) element by element at their tile, window and source-block edges,
in every form (window / dense x softmax on / off x collect / distribute x bf16 / bf16x3). Conventions and helpers as in
test_conv_edges_gpu.py, test_bn_edges_gpu.py and test_pool_resize_edges_gpu.py. u = 2^-24.

Reference. float64 on exactly what the kernels read: the fp32 logits A and the stored feat / dout / out (bf16, or
hi + lo, exact in fp32). The logit matrix L[t, s] (target t, source s) is built from an explicit index rule, checked
once against oracle.torch_oracle.psa_mask_torch in float64:
  window: the owner's entry idx = (oth_i - own_i + hh)*mW + (oth_j - own_j + hw), logit 0 outside the mask window;
  dense:  the owner's entry at the other pixel's flat position;
  owner = t, other = s for collect (L[t, s] = A[t, .]); owner = s, other = t for distribute.
Where a kernel consumes an earlier kernel's output the reference uses that value, and the value has its own check: P is
exp(L - m)*inv with the forward's statistics (m, inv), read by the forward itself (the statistics it just wrote), by
the feature gradient and by the logit gradient; the logit gradient's D reads the kernel's stored `out`.

Bounds, each derived next to the kernel lines it comes from (psa_fused.cu):
  statistics  m = max_s L[t, s] is a max of fp32 values: bit-exact against the float64 max, window zeros included.
              1/sum against 1/S, S = sum_s exp(L - m) in float64: every term carries the __expf error e(x) (below), the
              sum its fp32 adds and 1.f/sum one IEEE division (u):
                collect    one warp per row: ceil(Q/32) adds per lane + the 5-level shuffle tree: (ceil(Q/32) + 5)*u*S;
                distribute per warp an online sum over ceil(Q/8) sources, each step sum*__expf(m - mn) + __expf(l - mn)
                           (rescale error, product and add), then the merge of 8 partials with __expf(mk - m): with
                           R = m - min_s L[t, s] bounding every exponent, (6*ceil(Q/8) + 6.692*R + 13)*u*S;
                plus an absolute (Q + 16)*2^-126 for terms that ex2.approx.ftz flushes to zero.
  __expf      CUDA C++ Programming Guide (CUDA 12.9), Mathematical Functions, "Intrinsic Functions", single precision:
              __expf(x) has a maximum error of 2 + floor(abs(1.173*x)) ulp; one ulp is at most 2^-23 = 2u of the
              result. Its argument x = l - m is rounded once in fp32 (relative u, i.e. |x|*u on the result):
                e(x) = (2*(2 + floor(1.173*|x|)) + |x|)*u,  absolute floor 2^-126 (flushed results).
  P           pv = __expf(l - m)*inv: |pv - P| <= eP = P*(e(x) + u) + 2*2^-126 (the product's own rounding, the flush).
              Without softmax P = L exactly (eP = 0).
              bf16: the MMA reads bf16_rn(pv); rounding is monotone, so it lies between bf16(P - eP) and bf16(P + eP):
                the reference uses bf16(P) and the wider side of that bracket as the per-element P error (exact when
                no rounding boundary lies within eP, which is most elements).
              bf16x3: hi = bf16(pv), lo = bf16(pv - hi) made inside the kernel: |pv - hi - lo| <= 2^-16*|pv|, and the
                segment P_lo*B_lo that the three segments (P_hi*B_hi, P_lo*B_hi, P_hi*B_lo) leave out is at most
                2^-8*(1 + 2^-7)*|pv|*|B_lo|.
  out, dfeat  the wgmma chain over num_kb = ceil(Q/64) blocks of 64 sources (targets for dfeat) x 4 K-steps x nseg:
              steps = C_TRUNC*num_kb*4*nseg (the conv tests' truncation constant) + 1 for *scale, on
              S = scale*sum |P||B| (segments), plus scale*sum eP*|B| and the terms above; then the bf16 or hi/lo store
              through `ratio`.
  dattn       acc = sum_c dout*feat (K = C, segments): C_TRUNC*(C/64)*4*nseg steps on scale*sum |dout||feat|, and dP =
              scale*acc one rounding; D = sum_c dout*out_stored: one fmaf chain of C/4 channels per lane, then 2
              shuffle adds, (C/4 + 2)*u*sum |dout||out|; dL = pv*(dP - D): two more roundings, and eP*|dP - D|.
              Without softmax dL = dP.
  D           D is taken on the stored `out`, a design approximation of sum_s P*dP: |D - sum_s P*dP| is measured and
              held to sum_c |dout|*(the forward's bound on that element, storage included).
  composition every output is also checked against float64 autograd of test_psa_variants_gpu._composition on the
              stored operands (exact softmax, exact D), with the per-kernel bound plus the statistics' relative bound
              times P, the D bound, and the bf16x3 dout_lo*feat_lo product the kernel leaves out.

Teeth. Each case recomputes a reference without the contribution it guards and asserts that the same bound flags an
element: the last (partial) K block of 64 sources (forward) or targets (dfeat) ["kblock"]; the out-of-window logit-0
sources excluded instead of counted as 0 ["window0": from the statistics' sum and from the contraction]; collect and
distribute swapped, P from L^T ["transpose"]; the last row of the last (partial) tile ["lastrow"]; the P_lo*B_hi
segment in bf16x3 ["x3lo"]; in the distribute statistics, the sources of the last worker warp ["lastwarp"]; in the
logit gradient the D term ["D"] and the last 256-source block ["sblock"].

Geometry. psa_tile_rows is mirrored from the device's SM count: forward tiles psa_tile_rows(N, Q, 64, 1) rows (8 to 64),
logit-gradient tiles psa_tile_rows(N, Q, 128, ceil(Q/256)) rows over ceil(Q/256) source blocks; each case asserts the
branch it names and prints the statistics path (collect: one warp per row; distribute: 8 warps, online) and the P-fill
path (row-owner, or k-owner with its 32-row groups).

Hygiene, every case: a second call gives the same bits (out, stats, dfeat, dattn); the inputs are unchanged; out and
dfeat written through the C entry point at out_pitch 576 leave the padding channels at their sentinel; feat / dout /
out read as a channel slice at pitch 576 give the same bits; attn at an a_pitch wider than the mask with NaN padding
gives the same bits, and dattn's padding columns are exactly 0; in the window form dattn is exactly 0 at every entry
no (target, source) pair maps to; in the dense form with a_pitch == H*W (no memset in the entry point) a NaN-prefilled
dattn is fully overwritten.
"""
import ctypes
import zlib

import pytest
import torch

from oracle.torch_oracle import psa_mask_torch
from tests.test_bn_edges_gpu import SENTINEL
from tests.test_conv_edges_gpu import C_TRUNC, R_BF16, R_SPLIT, U, _act, _segments, cdiv, planes, ratio, report, stored
from tests.test_psa_variants_gpu import _composition

pytestmark = pytest.mark.gpu

DEV = "cuda"
C = 512
PITCH = 576                      # the padded pitch of the hygiene checks
TINY = 2.0 ** -126               # smallest normal fp32: ex2.approx.ftz flushes below it
EXPF_ULP, EXPF_SLOPE = 2.0, 1.173


@pytest.fixture(scope="module", autouse=True)
def _device():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.backends.cuda.matmul.allow_tf32 = False
    yield


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def tile_rows(n, q, max_rows, blocks_per_tile):
    """csrc/psa_fused.cu::psa_tile_rows."""
    want = n * q * blocks_per_tile // _sms()
    return max_rows if want >= max_rows else max(8, want)


def bound_ratio(out, ref, bound):
    """max |out - ref| / bound for an absolute per-element bound (`ratio` with r_out = 0 and one step)."""
    return ratio(out, ref, bound / U, 0.0, 1)


def bf16(x):
    return x.float().bfloat16().double()


# ------------------------------------------------------------------------------------------------ logit matrix
def owner_index(h, w, mh, mw, dense):
    """(idx, inside) [Q, Q] over (owner, other): the owner's attention entry for the other pixel."""
    q = h * w
    t = torch.arange(q, device=DEV)
    if dense:
        return t[None, :].expand(q, q), torch.ones((q, q), dtype=torch.bool, device=DEV)
    ti, tj = t // w, t % w
    a = ti[None, :] - ti[:, None] + (mh - 1) // 2
    b = tj[None, :] - tj[:, None] + (mw - 1) // 2
    inside = (a >= 0) & (a < mh) & (b >= 0) & (b < mw)
    return torch.where(inside, a * mw + b, 0), inside


def owner_gather(a, idx, inside):
    """G[n, own, oth] = a[n, own, idx[own, oth]], 0 outside the window; a [N, Q, a_pitch]."""
    g = torch.gather(a, 2, idx.expand(a.shape[0], -1, -1))
    return torch.where(inside, g, torch.zeros((), dtype=g.dtype, device=g.device))


def to_ts(g, psa_type):
    """(owner, other) -> (target, source): collect owns by the target, distribute by the source."""
    return g if psa_type == 0 else g.transpose(1, 2)


def exp_err(x):
    """Relative error of __expf(fl(x)) (module docstring)."""
    return (2 * (EXPF_ULP + torch.floor(EXPF_SLOPE * x.abs())) + x.abs()) * U


def softmax64(L):
    return torch.softmax(L, dim=-1)


# ------------------------------------------------------------------------------------------------ aggregation bound
def agg_terms(Pm, eP, Bp, scale):
    """(ref, S, extra) of out[r, c] = scale * sum_k P[r, k] * B[k, c] as the kernel forms it (module docstring).
    Pm, eP [N, R, K]; Bp = planes of B [N, K, C]."""
    eP = eP * (1 + 2.0 ** -10)
    if len(Bp) == 1:
        B = Bp[0]
        pc = bf16(Pm)
        width = torch.maximum(bf16(Pm + eP) - pc, pc - bf16(Pm - eP))
        return scale * (pc @ B), scale * (pc.abs() @ B.abs()), scale * (width @ B.abs())
    bh, bl = Bp
    pa = Pm.abs() + eP
    s = scale * ((pa * (1 + 2.0 ** -7)) @ (bh.abs() + bl.abs()))
    extra = scale * ((eP + 2.0 ** -16 * pa) @ (bh + bl).abs() + 2.0 ** -8 * (1 + 2.0 ** -7) * (pa @ bl.abs()))
    return scale * (Pm @ (bh + bl)), s, extra


def agg_ref(Pm, Bp, scale):
    """The same reference for a modified P (teeth): bf16(P) in bf16 mode, P itself in bf16x3."""
    if len(Bp) == 1:
        return scale * (bf16(Pm) @ Bp[0])
    return scale * (Pm @ (Bp[0] + Bp[1]))


def agg_ratio(out, ref, s, extra, steps, split):
    """`ratio` with the absolute P terms folded into the accumulation term: bound = steps*u*s + extra (+ storage)."""
    return ratio(out, ref, s + extra / (steps * U), R_SPLIT if split else R_BF16, steps)


def agg_bound(out, s, extra, steps, split):
    """The per-element bound of agg_ratio with its storage term (bf16: 2^-8*|out| covers the half gap)."""
    return steps * U * s + extra + (2.0 ** -16 * 1.01 if split else 2.0 ** -8) * out.abs()


# ------------------------------------------------------------------------------------------------ cases
# id: (N, H, W, mH, mW, dense, extra logit columns, softmax, logit regime, teeth, options). Regimes: randn2 = randn*2,
# sat = randn*30 (rows saturate, most P underflow), const = 0.75 everywhere (uniform P in the dense form), ties =
# round(randn*1.5) (exact ties at the row max), signed = randn (softmax-free logits of both signs). Options: grad_c
# (the logit gradient at another C), tile / gtile (the forward / logit-gradient tile branch the case exists for).
CASES = {
    # forward tiles
    "tile8-floor-q6": (1, 2, 3, 3, 5, False, 0, True, "randn2", ("transpose", "lastrow"), dict(tile="floor")),
    "tile13-odd-partial-q900": (2, 30, 30, 25, 31, False, 0, True, "randn2", ("kblock", "window0", "lastrow"),
                                dict(tile="odd-partial", gtile="le64")),
    "tile64-last1-q4225": (2, 65, 65, 9, 9, False, 0, True, "randn2", ("kblock", "window0", "lastrow", "sblock"),
                           dict(tile="last1", gtile="128")),
    "tile64-last41-kowner": (8, 45, 45, 31, 41, False, 0, True, "randn2", ("kblock", "lastrow", "sblock"),
                             dict(tile="last41", gtile="128")),
    "tile64-full-q1024-dense": (16, 32, 32, 32, 32, True, 0, True, "randn2", ("kblock", "transpose", "lastrow"),
                                dict(tile="full", gtile="128")),
    # sources
    "q25-idle-lanes": (1, 5, 5, 5, 5, False, 0, True, "randn2", ("window0", "transpose", "lastrow")),
    "q1": (1, 1, 1, 1, 1, False, 0, True, "randn2", ("lastrow",)),
    "q1-nosoftmax": (1, 1, 1, 1, 1, True, 3, False, "signed", ("lastrow",)),
    # logit gradient
    "grad-tile81-q900": (3, 30, 30, 59, 59, False, 0, True, "randn2", ("transpose", "sblock", "lastrow"),
                         dict(gtile="65-127")),
    "grad-q256-one-block": (1, 16, 16, 31, 31, False, 0, True, "randn2", ("transpose", "lastrow")),
    "grad-q257-w1": (1, 257, 1, 513, 1, False, 0, True, "randn2", ("transpose", "sblock", "kblock")),
    "grad-c64": (2, 9, 11, 9, 13, False, 0, True, "randn2", ("transpose", "lastrow"), dict(grad_c=64)),
    "grad-c192-dense": (2, 9, 11, 9, 11, True, 5, True, "randn2", ("transpose", "kblock"), dict(grad_c=192)),
    # maps and masks
    "w128": (1, 2, 128, 3, 129, False, 0, True, "randn2", ("window0", "kblock", "lastrow")),
    "h1": (1, 1, 100, 1, 61, False, 0, True, "randn2", ("window0", "kblock", "lastrow")),
    "mask-larger-than-map": (1, 6, 5, 15, 13, False, 4, True, "randn2", ("transpose", "lastrow")),
    "mask-1x1": (2, 7, 9, 1, 1, False, 0, True, "randn2", ("window0", "kblock", "lastrow")),
    "dense-nonsquare-mask-pitch": (2, 6, 7, 3, 14, True, 10, True, "randn2", ("transpose", "lastrow")),
    # the real shapes
    "psanet50-465-473": (16, 30, 30, 59, 59, False, 0, True, "randn2", ("transpose", "kblock", "sblock")),
    "cityscapes-713": (2, 45, 45, 89, 89, False, 0, True, "randn2", ("kblock", "sblock", "lastrow")),
    "compact-465": (2, 30, 30, 30, 30, True, 0, True, "randn2", ("transpose", "kblock", "lastrow")),
    # logit regimes
    "saturated": (2, 13, 11, 25, 21, False, 0, True, "sat", ("transpose",)),
    "constant-dense": (2, 9, 9, 9, 9, True, 0, True, "const", ("kblock", "lastrow")),
    "ties": (1, 8, 12, 15, 23, False, 0, True, "ties", ("transpose", "lastrow")),
    "nosoftmax-window": (2, 9, 12, 9, 7, False, 0, False, "signed", ("transpose", "kblock", "lastrow")),
    "nosoftmax-dense-pitch": (2, 13, 9, 13, 9, True, 6, False, "signed", ("transpose", "kblock")),
}

PARAMS = [pytest.param(name, psa_type, split, id="%s-%s-%s" % (name, ("collect", "distribute")[psa_type],
                                                                 "x3" if split else "bf16"))
          for name in CASES for psa_type in (0, 1) for split in (False, True)]


def _seed(name):
    return zlib.crc32(name.encode()) % 100000


def logits(shape, regime, gen):
    x = torch.randn(shape, device=DEV, generator=gen)
    return {"randn2": x * 2, "sat": x * 30, "const": torch.full_like(x, 0.75), "ties": torch.round(x * 1.5),
            "signed": x}[regime]


def _form(dense, softmax):
    from semseg_b200 import _lib
    return (_lib.PSA_DENSE if dense else 0) | (0 if softmax else _lib.PSA_NO_SOFTMAX)


def _p(t):
    return ctypes.c_void_p(t.data_ptr() if t is not None else 0)


def _ex_attend(mode, psa_type, form, attn, a_pitch, src, src_pitch, stats, dst, dst_pitch, geom, scale):
    from semseg_b200 import _lib, ops
    n, h, w, mh, mw = geom
    _lib.check(_lib.load().semseg_psa_attend_ex(mode, psa_type, form, _p(attn), a_pitch, _p(src), ops._lo(src),
                                                src_pitch, _p(stats), _p(dst), ops._lo(dst), dst_pitch, n, h, w, mh, mw,
                                                C, scale, ops._stream()), "semseg_psa_attend_ex")


def _ex_grad(psa_type, form, attn, a_pitch, stats, feat, out, dout, dattn, geom, scale, c):
    from semseg_b200 import _lib, ops
    n, h, w, mh, mw = geom
    pitch = lambda t: ops._nhwc_meta(t)[4] if t is not None else c      # noqa: E731
    _lib.check(_lib.load().semseg_psa_attend_bwd_attn_ex(psa_type, form, _p(attn), a_pitch, _p(stats), _p(feat),
                                                         ops._lo(feat), pitch(feat), _p(out), ops._lo(out), pitch(out),
                                                         _p(dout), ops._lo(dout), pitch(dout), _p(dattn), n, h, w, mh,
                                                         mw, c, scale, ops._stream()), "semseg_psa_attend_bwd_attn_ex")


def _padded(t, width, off=0):
    """A copy of activation t as channels [off, off + C) of a `width`-wide buffer (sentinel elsewhere)."""
    from semseg_b200 import ops
    buf = ops.empty_act(tuple(t.shape[-4:-1]) + (width,), t.dim() == 5, DEV).fill_(SENTINEL)
    view = buf[..., off:off + t.shape[-1]]
    view.copy_(t)
    return buf, view


# ------------------------------------------------------------------------------------------------ the test
@pytest.mark.parametrize("name,psa_type,split", PARAMS)
def test_psa_attend_element_bound(name, psa_type, split):
    from semseg_b200 import ops
    n, h, w, mh, mw, dense, pad, softmax, regime, teeth_names, o = (CASES[name] + ({},))[:11]
    q, nseg = h * w, 3 if split else 1
    gc = o.get("grad_c", C)
    scale = 1.0 / 3.0
    geom = (n, h, w, mh, mw)
    gen = torch.Generator(device=DEV).manual_seed(_seed(name) + 10 * psa_type + int(split))
    a_pitch = mh * mw + pad
    attn = logits((n, h, w, a_pitch), regime, gen)
    feat = _act(torch.relu(torch.randn((n, h, w, C), device=DEV, generator=gen)), split)
    dout = _act(torch.randn((n, h, w, C), device=DEV, generator=gen), split)
    inputs = [t.clone() for t in (attn, feat, dout)]
    claims = []

    # ---- geometry, tied to psa_tile_rows
    tr, nb = tile_rows(n, q, 64, 1), cdiv(q, 256)
    gtr = tile_rows(n, q, 128, nb)
    num_kb = cdiv(q, 64)
    last_tile = q - (cdiv(q, tr) - 1) * tr
    want = {"floor": tr == 8 and n * q < 8 * _sms(), "odd-partial": tr % 2 == 1 and q % tr != 0,
            "last1": tr == 64 and last_tile == 1, "last41": tr == 64 and 33 <= last_tile <= 63,
            "full": tr == 64 and q % 64 == 0 and last_tile == 64}
    if "tile" in o:
        assert want[o["tile"]], "forward tile %d rows, last tile %d: not the '%s' branch" % (tr, last_tile, o["tile"])
    gwant = {"128": gtr == 128, "le64": gtr <= 64, "65-127": 64 < gtr < 128}
    if "gtile" in o:
        assert gwant[o["gtile"]], "logit-gradient tile %d rows: not the '%s' branch" % (gtr, o["gtile"])
    claims.append("fwd tile %d rows (last %d), logit-grad tile %d rows x %d source block(s) (last %d)" %
                  (tr, last_tile, gtr, nb, q - 256 * (nb - 1)))
    row_owner_fwd = psa_type == 0
    claims.append("P fill fwd %s / dfeat %s" % ("row-owner" if row_owner_fwd else "k-owner (%d row group(s))" %
                                                cdiv(min(tr, last_tile), 32), "k-owner" if row_owner_fwd else
                                                "row-owner"))
    if softmax:
        claims.append("stats %s" % ("collect, one warp per row" + (", %d idle lanes" % (32 - q) if q < 32 else "")
                                    if psa_type == 0 else "distribute, 8 warps x %d sources%s" %
                                    (cdiv(q, 8), ", %d empty warp(s)" % (8 - cdiv(q, cdiv(q, 8))) if q < 8 else "")))
    if name == "grad-q257-w1":
        assert q == 257 and nb == 2
    if name == "grad-q256-one-block":
        assert q == 256 and nb == 1
    if name.startswith("psanet50"):
        assert nb == 4 and a_pitch == 3481

    # ---- kernels, twice
    def run():
        out, stats = ops.psa_attend(attn, feat, psa_type, mh, mw, scale, compact=dense, softmax=softmax)
        dfeat, _ = ops.psa_attend(attn, dout, psa_type, mh, mw, scale, stats=stats, mode=1, compact=dense,
                                  softmax=softmax)
        return out, stats, dfeat

    out, stats, dfeat = run()
    out2, stats2, dfeat2 = run()
    assert torch.equal(out, out2) and torch.equal(dfeat, dfeat2), "forward / dfeat not bit-identical on a second call"
    assert stats is None or torch.equal(stats, stats2)
    if gc == C:
        gfeat, gdout, gout = feat, dout, out
    else:                                   # the logit gradient at another C: its own operands, the forward's stats
        gfeat = _act(torch.relu(torch.randn((n, h, w, gc), device=DEV, generator=gen)), split)
        gdout = _act(torch.randn((n, h, w, gc), device=DEV, generator=gen), split)
        gout = _act(torch.randn((n, h, w, gc), device=DEV, generator=gen), split)
        claims.append("logit gradient at C = %d (D: %d channels per lane)" % (gc, gc // 4))
    dattn = ops.psa_attend_bwd_attn(attn, stats, gfeat, gout if softmax else None, gdout, psa_type, mh, mw, scale,
                                    compact=dense, softmax=softmax)
    dattn2 = ops.psa_attend_bwd_attn(attn, stats, gfeat, gout if softmax else None, gdout, psa_type, mh, mw, scale,
                                     compact=dense, softmax=softmax)
    assert torch.equal(dattn, dattn2), "dattn not bit-identical on a second call"
    for a, b in zip(inputs, (attn, feat, dout)):
        assert torch.equal(a, b), "an input was modified"

    # ---- the logit matrix and P
    idx, inside_o = owner_index(h, w, mh, mw, dense)
    A = attn.double().reshape(n, q, a_pitch)
    L = to_ts(owner_gather(A, idx, inside_o), psa_type)
    inside = to_ts(inside_o[None].expand(n, -1, -1), psa_type)
    worst, teeth = {}, {}
    if softmax:
        m_k, inv_k = stats[..., 0].double(), stats[..., 1].double()
        assert torch.equal(m_k, L.max(-1).values), "row max differs from the float64 max of the stored logits"
        x = L - m_k[..., None]
        e = torch.exp(x)
        S = e.sum(-1)
        if psa_type == 0:
            chain = (cdiv(q, 32) + 5) * U
        else:
            chain = (6 * cdiv(q, 8) + 6.692 * (m_k - L.min(-1).values) + 13) * U
        rel_inv = ((e * exp_err(x)).sum(-1) + chain * S + (q + 16) * TINY) / S + U
        inv_b = rel_inv / S
        worst["stats"] = bound_ratio(inv_k, 1 / S, inv_b)
        P = e * inv_k[..., None]
        eP = P * (exp_err(x) + U) + 2 * TINY
    else:
        rel_inv = torch.zeros((n, q), dtype=torch.float64, device=DEV)
        P, eP = L, torch.zeros_like(L)

    def p_of(Lm):
        return softmax64(Lm) if softmax else Lm

    # ---- forward and dfeat
    fp, dp = planes(feat, split), planes(dout, split)
    fp = [t.reshape(n, q, C) for t in fp]
    dp = [t.reshape(n, q, C) for t in dp]
    steps = C_TRUNC * num_kb * 4 * nseg + 1
    out_s, dfeat_s = stored(out).reshape(n, q, C), stored(dfeat).reshape(n, q, C)
    PT, ePT = P.transpose(1, 2), eP.transpose(1, 2)
    fref, fS, fX = agg_terms(P, eP, fp, scale)
    dref, dS, dX = agg_terms(PT, ePT, dp, scale)
    worst["out"] = agg_ratio(out_s, fref, fS, fX, steps, split)
    worst["dfeat"] = agg_ratio(dfeat_s, dref, dS, dX, steps, split)

    def agg_teeth(label, Pt, rowcut=False, k0=None):
        for key, Pm, Bp, o_s, S_, X_ in (("out", Pt, fp, out_s, fS, fX), ("dfeat", Pt.transpose(1, 2), dp, dfeat_s,
                                                                           dS, dX)):
            if k0 is not None:
                Pm = Pm.clone()
                Pm[..., k0:] = 0
            r = agg_ref(Pm, Bp, scale)
            if rowcut:
                r = r.clone()
                r[-1, -1] = 0
            teeth["%s/%s" % (label, key)] = agg_ratio(o_s, r, S_, X_, steps, split)

    # ---- logit gradient
    gfp = [t.reshape(n, q, gc) for t in planes(gfeat, split)]
    gdp = [t.reshape(n, q, gc) for t in planes(gdout, split)]
    acc = sacc = 0
    for da, fa in _segments(gdp, gfp):
        acc = acc + da @ fa.transpose(1, 2)
        sacc = sacc + da.abs() @ fa.abs().transpose(1, 2)
    gsteps = C_TRUNC * (gc // 64) * 4 * nseg
    dP = scale * acc
    E = scale * gsteps * U * sacc + U * dP.abs()
    gdo = stored(gdout).reshape(n, q, gc)
    if softmax:
        go = stored(gout).reshape(n, q, gc)
        D = (gdo * go).sum(-1)
        E = E + ((gc / 4 + 2) * U * (gdo.abs() * go.abs()).sum(-1))[..., None]
        diff = dP - D[..., None]
        gref = P * diff
        gb = eP * (diff.abs() + E) + P.abs() * (E + 2 * U * diff.abs()) + TINY
    else:
        gref, gb = dP, E
    dA = dattn.double().reshape(n, q, a_pitch)
    gk = to_ts(owner_gather(dA, idx, inside_o), psa_type)
    zero = torch.zeros((), dtype=torch.float64, device=DEV)
    gref, gb = torch.where(inside, gref, zero), torch.where(inside, gb, zero)
    worst["dattn"] = bound_ratio(gk, gref, gb)

    def grad_teeth(label, r):
        teeth["%s/dattn" % label] = bound_ratio(gk, torch.where(inside, r, zero), gb)

    # ---- teeth
    names = list(teeth_names)
    if split and regime != "sat" and q > 1:
        names.append("x3lo")
    if softmax:
        names.append("D")
        if psa_type == 1 and 7 * cdiv(q, 8) < q:
            names.append("lastwarp")
    for t in names:
        if t == "kblock":
            agg_teeth(t, P, k0=64 * (num_kb - 1))
            claims.append("teeth kblock: %s [%d, %d) dropped" % ("sources / targets", 64 * (num_kb - 1), q))
        elif t == "lastrow":
            agg_teeth(t, P, rowcut=True)
            if q > 1 or not softmax:         # Q = 1: P = 1 and D = dP, the only logit gradient is 0
                r = gref.clone()
                r[-1, -1] = 0
                grad_teeth(t, r)
        elif t == "window0":
            assert not bool(inside.all()), "window0 needs out-of-window sources"
            agg_teeth(t, torch.where(inside, P, zero))
            if softmax:
                teeth["window0/stats"] = bound_ratio(inv_k, 1 / (e * inside).sum(-1), inv_b)
        elif t == "transpose":
            Lt = L.transpose(1, 2)
            Pt = p_of(Lt)
            agg_teeth(t, Pt)
            # the swapped kernel writes its (t, s) value at the entry this orientation reads for (s, t)
            grad_teeth(t, (Pt * diff if softmax else dP).transpose(1, 2))
            if softmax:
                teeth["transpose/stats"] = bound_ratio(inv_k, 1 / torch.exp(Lt - Lt.max(-1, keepdim=True).values)
                                                       .sum(-1), inv_b)
        elif t == "x3lo":
            agg_teeth(t, bf16(P))
        elif t == "lastwarp":
            q0 = 7 * cdiv(q, 8)
            teeth["lastwarp/stats"] = bound_ratio(inv_k, 1 / e[..., :q0].sum(-1), inv_b)
        elif t == "D":
            grad_teeth(t, P * dP)
        elif t == "sblock":
            assert nb > 1
            r = gref.clone()
            r[..., 256 * (nb - 1):] = 0
            grad_teeth(t, r)
        else:
            raise AssertionError(t)

    # ---- D: the design approximation, measured
    if softmax and gc == C:
        fb = agg_bound(out_s, fS, fX, steps, split)
        d_exact = (gdo * fref).sum(-1)
        d_err = (D - d_exact).abs()
        d_bound = (gdo.abs() * fb).sum(-1)
        d_rel = float((d_err / (gdo.abs() * go.abs()).sum(-1).clamp_min(1e-300)).max())
        worst["D"] = float((d_err / d_bound).max())
        claims.append("D on stored out vs sum_s P*dP: max |dD| / sum|dout*out| = %.3g" % d_rel)

    # ---- float64 autograd of the reference composition
    ar = A.reshape(n, h, w, a_pitch).clone().requires_grad_(True)
    fr = stored(feat).clone().requires_grad_(True)
    comp = _composition(ar, fr, psa_type, mh, mw, scale, dense, softmax)
    comp.backward(stored(dout))
    lolo_f = 0 if not split else scale * (dp[1].abs() @ fp[1].abs().transpose(1, 2))
    if gc == C:
        Pex = p_of(L)
        crel = rel_inv[..., None] * P
        if not split:                        # the composition's P is not rounded to bf16
            crel = crel + (bf16(P) - P).abs()
        cX = fX + scale * (crel @ sum(t.abs() for t in fp))
        worst["composition/out"] = agg_ratio(out_s, comp.detach().reshape(n, q, C), fS, cX, steps, split)
        cdX = dX + scale * (crel.transpose(1, 2) @ sum(t.abs() for t in dp))
        worst["composition/dfeat"] = agg_ratio(dfeat_s, fr.grad.reshape(n, q, C), dS, cdX, steps, split)
        cg = to_ts(owner_gather(ar.grad.reshape(n, q, a_pitch), idx, inside_o), psa_type)
        cb = gb + lolo_f
        if softmax:
            fbc = agg_bound(out_s, fS, cX, steps, split)
            cb = cb + crel * diff.abs() + Pex * ((gdo.abs() * fbc).sum(-1)[..., None] + lolo_f)
        worst["composition/dattn"] = bound_ratio(gk, torch.where(inside, cg, zero), torch.where(inside, cb, zero))

    # ---- hygiene
    form = _form(dense, softmax)
    # out / dfeat through the C entry point at out_pitch 576
    for mode, src, want_t in ((0, feat, out), (1, dout, dfeat)):
        buf, view = _padded(want_t, PITCH)
        st = torch.empty_like(stats) if (softmax and mode == 0) else stats
        _ex_attend(mode, psa_type, form, attn, a_pitch, src, C, st, view, PITCH, geom, scale)
        assert torch.equal(view, want_t), "out_pitch %d changes the result" % PITCH
        assert bool((buf[..., C:].float() == SENTINEL).all()), "the padding channels lost their sentinel"
        if mode == 0 and softmax:
            assert torch.equal(st, stats)
    # feat / dout / out as channel slices at pitch 576
    fs, ds = _padded(feat, PITCH, 64)[1], _padded(dout, PITCH, 64)[1]
    o_sl, st_sl = ops.psa_attend(attn, fs, psa_type, mh, mw, scale, compact=dense, softmax=softmax)
    d_sl, _ = ops.psa_attend(attn, ds, psa_type, mh, mw, scale, stats=stats, mode=1, compact=dense, softmax=softmax)
    assert torch.equal(o_sl, out) and torch.equal(d_sl, dfeat) and (stats is None or torch.equal(st_sl, stats))
    gs = [_padded(t, PITCH + gc - C, 64)[1] for t in (gfeat, gout, gdout)]
    g_sl = ops.psa_attend_bwd_attn(attn, stats, gs[0], gs[1] if softmax else None, gs[2], psa_type, mh, mw, scale,
                                   compact=dense, softmax=softmax)
    assert torch.equal(g_sl, dattn), "channel slices at pitch %d change dattn" % PITCH
    # attn at a wider a_pitch, padding columns NaN
    aw = torch.full((n, h, w, a_pitch + 24), float("nan"), device=DEV)
    aw[..., :a_pitch] = attn
    o_w, st_w = ops.psa_attend(aw, feat, psa_type, mh, mw, scale, compact=dense, softmax=softmax)
    d_w, _ = ops.psa_attend(aw, dout, psa_type, mh, mw, scale, stats=st_w, mode=1, compact=dense, softmax=softmax)
    g_w = ops.psa_attend_bwd_attn(aw, st_w, gfeat, gout if softmax else None, gdout, psa_type, mh, mw, scale,
                                  compact=dense, softmax=softmax)
    assert torch.equal(o_w, out) and torch.equal(d_w, dfeat) and (stats is None or torch.equal(st_w, stats))
    assert torch.equal(g_w[..., :a_pitch], dattn) and bool((g_w[..., a_pitch:] == 0).all())
    # entries no (target, source) pair maps to are exactly zero; the dense form writes every entry
    if not dense:
        hit = torch.zeros((q, a_pitch), dtype=torch.int32, device=DEV)
        hit.scatter_add_(1, idx, inside_o.int())
        hit = hit > 0
        assert bool((dA[:, ~hit] == 0).all()), "dattn is not 0 outside every window"
        claims.append("%d of %d dattn entries outside every window: exactly 0" % (int((~hit).sum()), q * a_pitch))
    else:
        assert bool((dA[..., q:] == 0).all())
        if a_pitch == q:
            pre = torch.full_like(attn[..., :a_pitch], float("nan"))
            _ex_grad(psa_type, form, attn, a_pitch, stats, gfeat, gout if softmax else None, gdout, pre, geom, scale,
                     gc)
            assert not bool(pre.isnan().any()), "a (target, source) pair of the dense form was never written"
            assert torch.equal(pre, dattn)
            claims.append("dense, a_pitch == H*W: NaN-prefilled dattn fully overwritten")
    torch.cuda.synchronize()

    claims.append("worst " + ", ".join("%s %.3g" % kv for kv in worst.items()))
    tw = min(teeth, key=teeth.get)
    claims.append("teeth " + ", ".join("%s %.3g" % kv for kv in teeth.items()))
    for k, v in teeth.items():
        assert v > 1.0, "teeth %s: the bound cannot see the guarded contribution (%.3g)" % (k, v)
    report("%s-%s-%s" % (name, ("collect", "distribute")[psa_type], "x3" if split else "bf16"), claims,
           max(worst.values()), teeth[tw])


# ------------------------------------------------------------------------------------------------ index rule
@pytest.mark.parametrize("geom", [(2, 5, 7, 9, 13), (1, 6, 5, 3, 7), (1, 4, 4, 11, 9), (2, 3, 8, 1, 1)])
def test_index_rule_matches_psa_mask_torch(geom):
    """The window index rule of the references above, against oracle.torch_oracle.psa_mask_torch in float64 (tied to
    the reference's psamask by test_oracle_cpu.py), for both psa types; the dense rule against _composition's view."""
    n, h, w, mh, mw = geom
    q = h * w
    gen = torch.Generator(device=DEV).manual_seed(q)
    a = torch.randn((n, h, w, mh * mw), device=DEV, generator=gen, dtype=torch.float64)
    idx, inside = owner_index(h, w, mh, mw, False)
    for psa_type in (0, 1):
        L = to_ts(owner_gather(a.reshape(n, q, -1), idx, inside), psa_type)
        y = psa_mask_torch(a.permute(0, 3, 1, 2).contiguous(), psa_type, mh, mw)      # [n, source, target]
        assert torch.equal(L, y.reshape(n, q, q).transpose(1, 2))
    d = torch.randn((n, h, w, q), device=DEV, generator=gen, dtype=torch.float64)
    didx, dins = owner_index(h, w, h, w, True)
    for psa_type in (0, 1):
        L = to_ts(owner_gather(d.reshape(n, q, q), didx, dins), psa_type)
        eye = torch.eye(q, dtype=torch.float64, device=DEV).reshape(1, q, q).expand(n, q, q)
        # the composition with an identity feature map returns P^T columns: out[t, s] = P[t, s] without softmax
        y = _composition(d, eye.reshape(n, h, w, q), psa_type, h, w, 1.0, True, False)
        assert torch.equal(L, y.reshape(n, q, q))
