"""CPU tier for the fused attention entry points (csrc/psa_fused.cu: semseg_psa_attend_ex, semseg_psa_attend_bwd_attn_ex):
an operand the kernels would access out of line is SEMSEG_E_INVALID before any CUDA call and before any launch:
  * stats (read, and written by the forward, as float2) that is not 8-byte aligned;
  * the forward's out / out_lo (stored as bf16 pairs) that is not 4-byte aligned, feat / feat_lo (TMA) not 16-byte
    aligned;
  * in the logit gradient, feat, dout and out with a pitch below C (rows that overlap), out / out_lo (16-byte vector
    loads in the D term) not 16-byte aligned, and feat_lo / dout_lo not 16-byte aligned. The logit gradient clears
    dattn with a cudaMemsetAsync before its tensor-map encodes; every one of these checks runs ahead of it.
No GPU is needed: the pointers are fake and never dereferenced, because every call here fails validation."""
import ctypes

import pytest

from semseg_b200 import _lib

P = ctypes.c_void_p(1 << 20)        # 16-byte aligned, never dereferenced
C = 512
H = W = 3
M = 3                               # 3 x 3 window mask


def _off(k):
    return ctypes.c_void_p(P.value + k)


def _attend(mode=0, form=0, stats=P, feat=P, feat_lo=None, feat_pitch=C, out=P, out_lo=None, out_pitch=C):
    # semseg_psa_attend_ex(mode, psa_type, form, attn, a_pitch, feat, feat_lo, feat_pitch, stats, out, out_lo, out_pitch,
    #                      N, H, W, mH, mW, C, scale, stream)
    return _lib.load().semseg_psa_attend_ex(mode, 0, form, P, M * M, feat, feat_lo, feat_pitch, stats, out, out_lo,
                                            out_pitch, 1, H, W, M, M, C, ctypes.c_float(1.0), None)


def _attn_grad(form=0, stats=P, feat=P, feat_lo=None, feat_pitch=C, out=P, out_lo=None, out_pitch=C, dout=P,
               dout_lo=None, dout_pitch=C, c=C):
    # semseg_psa_attend_bwd_attn_ex(psa_type, form, attn, a_pitch, stats, feat, feat_lo, feat_pitch, out, out_lo,
    #                               out_pitch, dout, dout_lo, dout_pitch, dattn, N, H, W, mH, mW, C, scale, stream)
    return _lib.load().semseg_psa_attend_bwd_attn_ex(0, form, P, M * M, stats, feat, feat_lo, feat_pitch, out, out_lo,
                                                     out_pitch, dout, dout_lo, dout_pitch, P, 1, H, W, M, M, c,
                                                     ctypes.c_float(1.0), None)


def _rejected(call, *words):
    lib = _lib.load()
    before = _lib.launch_count()
    status = call()
    msg = lib.semseg_last_error()
    assert status == -1, (status, msg)          # SEMSEG_E_INVALID, not SEMSEG_E_CUDA from a CUDA call that ran first
    assert all(w.encode() in msg for w in words), msg
    assert _lib.launch_count() == before


FORWARD = {
    "stats-4-byte": (lambda: _attend(stats=_off(4)), ("stats", "8-byte aligned")),
    "stats-4-byte-dfeat": (lambda: _attend(mode=1, stats=_off(4)), ("stats", "8-byte aligned")),
    "out-2-byte": (lambda: _attend(out=_off(2)), ("4-byte aligned",)),
    "out_lo-2-byte": (lambda: _attend(feat_lo=P, out_lo=_off(6)), ("4-byte aligned",)),
    "feat-8-byte": (lambda: _attend(feat=_off(8)), ("16-byte aligned",)),
    "feat_lo-8-byte": (lambda: _attend(feat_lo=_off(8), out_lo=P), ("16-byte aligned",)),
}

LOGIT_GRAD = {
    "stats-4-byte": (lambda: _attn_grad(stats=_off(4)), ("stats", "8-byte aligned")),
    "feat-pitch-below-C": (lambda: _attn_grad(feat_pitch=C - 8), ("pitch 504 is smaller than C = 512",)),
    "out-pitch-below-C": (lambda: _attn_grad(out_pitch=C - 64), ("pitch 448 is smaller than C = 512",)),
    "dout-pitch-below-C": (lambda: _attn_grad(dout_pitch=56, c=64), ("pitch 56 is smaller than C = 64",)),
    "out-8-byte": (lambda: _attn_grad(out=_off(8)), ("16-byte aligned",)),
    "out_lo-8-byte": (lambda: _attn_grad(feat_lo=P, dout_lo=P, out_lo=_off(8)), ("16-byte aligned",)),
    "feat_lo-8-byte": (lambda: _attn_grad(feat_lo=_off(8), dout_lo=P, out_lo=P), ("16-byte aligned",)),
    "dout_lo-8-byte": (lambda: _attn_grad(feat_lo=P, dout_lo=_off(8), out_lo=P), ("16-byte aligned",)),
    "dense-feat-pitch-below-C": (lambda: _attn_grad(form=_lib.PSA_DENSE, feat_pitch=C - 8), ("smaller than C",)),
}


@pytest.mark.parametrize("name", list(FORWARD))
def test_psa_attend_rejects_misaligned_operands(name):
    call, words = FORWARD[name]
    _rejected(call, "psa_attend", *words)


@pytest.mark.parametrize("name", list(LOGIT_GRAD))
def test_psa_attend_bwd_attn_rejects_before_the_memset(name):
    call, words = LOGIT_GRAD[name]
    _rejected(call, "psa_attend_bwd_attn", *words)


def test_softmax_free_logit_gradient_does_not_check_the_unread_out():
    """Without softmax the logit gradient reads neither out nor stats: a misaligned out is not an error there (the call
    then fails later, on the fake dout pitch below)."""
    _rejected(lambda: _attn_grad(form=_lib.PSA_NO_SOFTMAX, stats=None, out=_off(8), dout_pitch=C - 8),
              "pitch 504 is smaller than C = 512")
