"""CPU tier for the BatchNorm and element-wise activation entry points of csrc/bn.cu: an operand those kernels would
access with misaligned 16-byte vectors (a hi or lo base that is not 16-byte aligned, e.g. the channel slice
buf[..., 4:68]) or whose rows overlap (pitch < C) is SEMSEG_E_INVALID before anything is launched. No GPU is needed:
the pointers are fake and never dereferenced, because every call here fails validation."""
import ctypes

import pytest

from semseg_b200 import _lib

P = ctypes.c_void_p(16)          # 16-byte aligned, never dereferenced
ODD = ctypes.c_void_p(18)        # 2-byte aligned: one bf16 channel into a buffer
HALF = ctypes.c_void_p(24)       # 8-byte aligned: a slice starting 4 channels into a buffer (buf[..., 4:68])
C = 64


def _lib_err():
    return _lib.load().semseg_last_error()


def _apply(x=P, x_lo=None, x_pitch=C, res=P, res_lo=None, res_pitch=C, y=P, y_lo=None, y_pitch=C):
    return _lib.load().semseg_bn_apply(x, x_lo, x_pitch, P, res, res_lo, res_pitch, y, y_lo, y_pitch, 100, C, 1, None)


def _bwd_reduce(dy=P, dy_lo=None, dy_pitch=C, y=P, y_lo=None, y_pitch=C, x=P, x_lo=None, x_pitch=C, relu=1,
                peers=None, world=1):
    lib = _lib.load()
    return lib.semseg_bn_bwd_reduce(dy, dy_lo, dy_pitch, y, y_lo, y_pitch, x, x_lo, x_pitch, P, P, 100, C, relu, P,
                                    lib.semseg_bn_workspace_floats(100, C), P, P, peers, world, 0, 0, 4 * C, P, None)


def _bwd_apply(dy=P, dy_lo=None, dy_pitch=C, y=P, y_lo=None, y_pitch=C, x=P, x_lo=None, x_pitch=C, dx=P, dx_lo=None,
               dx_pitch=C, dres=P, dres_lo=None, dres_pitch=C, relu=1):
    return _lib.load().semseg_bn_bwd_apply(dy, dy_lo, dy_pitch, y, y_lo, y_pitch, x, x_lo, x_pitch, P, P, P, P, 100.0,
                                           100, C, relu, dx, dx_lo, dx_pitch, dres, dres_lo, dres_pitch, P, None)


def _bwd_frozen(dy=P, dy_lo=None, dy_pitch=C, y=P, y_lo=None, y_pitch=C, raw=P, raw_lo=None, raw_pitch=C, d_raw=P,
                d_raw_lo=None, d_raw_pitch=C, dres=P, dres_lo=None, dres_pitch=C):
    return _lib.load().semseg_bn_bwd_frozen(dy, dy_lo, dy_pitch, y, y_lo, y_pitch, raw, raw_lo, raw_pitch, P, P, P, P,
                                            1e-5, 100, C, 1, d_raw, d_raw_lo, d_raw_pitch, dres, dres_lo, dres_pitch, P,
                                            1 << 30, P, None)


def _add(a=P, a_lo=None, a_pitch=C, b=P, b_lo=None, b_pitch=C, out=P, out_lo=None, out_pitch=C):
    return _lib.load().semseg_add_act(a, a_lo, a_pitch, b, b_lo, b_pitch, out, out_lo, out_pitch, 100, C, None)


def _scale(x=P, x_lo=None, x_pitch=C, scale=P, out=P, out_lo=None, out_pitch=C):
    return _lib.load().semseg_scale_nc(x, x_lo, x_pitch, scale, out, out_lo, out_pitch, 2, 50, C, None)


def _to_act(out=P, out_lo=None, out_pitch=C, c=C - 3, cp=C):
    return _lib.load().semseg_f32_to_act(P, c, out, out_lo, out_pitch, 100, c, cp, None)


def _to_f32(x=P, x_lo=None, x_pitch=C):
    return _lib.load().semseg_act_to_f32(x, x_lo, x_pitch, P, C, 100, C, None)


# (entry point, name in the message, the activation operands it reads or writes with 16-byte vectors: (hi, lo, pitch))
CALLS = [
    (_apply, "bn_apply", [("x", "x_lo", "x_pitch"), ("res", "res_lo", "res_pitch"), ("y", "y_lo", "y_pitch")]),
    (_bwd_reduce, "bn_bwd_reduce", [("dy", "dy_lo", "dy_pitch"), ("y", "y_lo", "y_pitch"), ("x", "x_lo", "x_pitch")]),
    (_bwd_apply, "bn_bwd_apply", [("dy", "dy_lo", "dy_pitch"), ("y", "y_lo", "y_pitch"), ("x", "x_lo", "x_pitch"),
                                  ("dx", "dx_lo", "dx_pitch"), ("dres", "dres_lo", "dres_pitch")]),
    (_bwd_frozen, "bn_bwd_frozen", [("dy", "dy_lo", "dy_pitch"), ("y", "y_lo", "y_pitch"),
                                    ("raw", "raw_lo", "raw_pitch"), ("d_raw", "d_raw_lo", "d_raw_pitch"),
                                    ("dres", "dres_lo", "dres_pitch")]),
    (_add, "add_act", [("a", "a_lo", "a_pitch"), ("b", "b_lo", "b_pitch"), ("out", "out_lo", "out_pitch")]),
    (_scale, "scale_nc", [("x", "x_lo", "x_pitch"), ("out", "out_lo", "out_pitch")]),
    (_to_act, "f32_to_act", [("out", "out_lo", "out_pitch")]),
    (_to_f32, "act_to_f32", [("x", "x_lo", "x_pitch")]),
]
IDS = [c[1] for c in CALLS]


def _split(names):
    """Keyword arguments that make every activation operand of the call split (lo planes at an aligned address)."""
    return {lo: P for _, lo, _ in names}


def _rejected(call, name, what, **kw):
    lib = _lib.load()
    before = lib.semseg_launch_count()
    assert call(**kw) == -1, kw
    msg = _lib_err()
    assert name.encode() in msg and what.encode() in msg, (kw, msg)
    assert lib.semseg_launch_count() == before, "a rejected call launched a kernel"


@pytest.mark.parametrize("call,name,operands", CALLS, ids=IDS)
def test_misaligned_base_rejected_before_launch(call, name, operands):
    """Each operand in turn at a 2-byte and an 8-byte aligned base, plain and split; in split storage also the lo plane
    alone (a hi plane that is aligned does not make the lo plane aligned)."""
    for hi, lo, _ in operands:
        for bad in (ODD, HALF):
            _rejected(call, name, "aligned", **{hi: bad})
            _rejected(call, name, "aligned", **dict(_split(operands), **{hi: bad}))
            _rejected(call, name, "aligned", **dict(_split(operands), **{lo: bad}))


@pytest.mark.parametrize("call,name,operands", CALLS, ids=IDS)
def test_pitch_below_channels_rejected_before_launch(call, name, operands):
    """A pitch that is a multiple of 8 but smaller than C (the width the kernel writes for f32_to_act: Cp) would make
    rows overlap."""
    for _, _, pitch in operands:
        _rejected(call, name, "pitch", **{pitch: C - 8})


def test_scale_nc_misaligned_scale_rejected():
    """scale_nc reads its fp32 [N][C] factors as float4 pairs."""
    for bad in (ctypes.c_void_p(20), HALF):
        _rejected(_scale, "scale_nc", "aligned", scale=bad)


def test_operands_the_kernel_does_not_touch_are_not_checked():
    """y is read only for the ReLU mask: without ReLU an unaligned y is never dereferenced, so the call is judged on its
    other operands (here it is rejected for the misaligned x at 0x18, not for y at 0x12)."""
    for call, name in ((_bwd_reduce, "bn_bwd_reduce"), (_bwd_apply, "bn_bwd_apply")):
        _rejected(call, name, "0x18", relu=0, y=ODD, x=HALF)


def test_slices_on_eight_channel_boundaries_pass_the_check():
    """What the networks pass: channel slices that start at a multiple of 8 channels (16 bytes) of a split buffer, with
    the lo plane behind the hi plane, pitch > C. The call gets past the alignment and pitch check and is stopped by the
    next one (a bad peer table), so nothing is launched."""
    m, width = 100, 4 * C + 16
    plane = 2 * m * width                      # bytes per plane of a [M][width] bf16 buffer
    base = 1 << 20
    kw = {}
    for k, (hi, lo, pitch) in enumerate((("dy", "dy_lo", "dy_pitch"), ("y", "y_lo", "y_pitch"),
                                         ("x", "x_lo", "x_pitch"))):
        off = 2 * 8 * (k + 1)                  # channels 8, 16, 24 of the buffer
        kw.update({hi: ctypes.c_void_p(base + off), lo: ctypes.c_void_p(base + plane + off), pitch: width})
    peers = (ctypes.c_void_p * 8)(*([16] * 8))
    _rejected(_bwd_reduce, "world 9", "world", peers=peers, world=9, **kw)
