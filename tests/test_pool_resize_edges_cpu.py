"""CPU tier for the pyramid-pooling (csrc/ppm.cu), bilinear-resize (csrc/resize.cu), max-pool (csrc/pool.cu) and
stride-2 layout (csrc/layout.cu: space_to_phases, phases_to_space, im2col3x3s2) entry points: an operand those kernels
would access with misaligned vectors (a hi or lo base that is not 16-byte aligned, e.g. the channel slice
buf[..., 4:68]; an argcode or im2col input that is not 8-byte aligned for its uint2 accesses), whose rows overlap
(pitch < C), or whose channel slice runs past the pitch (ppm_upsample_bwd's c_off + nb*Cr) is SEMSEG_E_INVALID before
anything is launched. No GPU is needed: the pointers are fake and never dereferenced, because every call here fails
validation."""
import ctypes

import pytest

from semseg_b200 import _lib

P = ctypes.c_void_p(16)          # 16-byte aligned, never dereferenced
ODD = ctypes.c_void_p(18)        # 2-byte aligned: one bf16 channel into a buffer
HALF = ctypes.c_void_p(24)       # 8-byte aligned: a slice starting 4 channels into a buffer (buf[..., 4:68])
C = 64
BINS = (1, 2, 3, 6)
NB = len(BINS)


def _bins():
    return (ctypes.c_int * NB)(*BINS)


def _ptrs(v):
    """A per-bin pointer table with every bin at `v`."""
    return (ctypes.c_void_p * NB)(*([v.value] * NB))


def _pool(x=P, x_lo=None, x_pitch=C, bin_ptr=P, bin_lo=None):
    lo = _ptrs(bin_lo) if x_lo is not None else None
    return _lib.load().semseg_ppm_pool(x, x_lo, x_pitch, 2, 9, 12, C, _bins(), _ptrs(bin_ptr), lo, NB, None)


def _pool_bwd(dx=P, dx_lo=None, dx_pitch=C, add=P, add_lo=None, add_pitch=C + NB * 8, bin_ptr=P, bin_lo=None):
    lo = _ptrs(bin_lo) if dx_lo is not None else None
    return _lib.load().semseg_ppm_pool_bwd(_ptrs(bin_ptr), lo, _bins(), NB, 2, 9, 12, C, dx, dx_lo, dx_pitch, add,
                                           add_lo, add_pitch, None)


def _up(x=P, x_lo=None, x_pitch=C, out=P, out_lo=None, out_pitch=C + NB * 8, bin_ptr=P, bin_lo=None):
    lo = _ptrs(bin_lo) if x_lo is not None else None
    return _lib.load().semseg_ppm_upsample_concat(x, x_lo, x_pitch, _ptrs(bin_ptr), lo, _bins(), NB, 2, 9, 12, C,
                                                  8, out, out_lo, out_pitch, None)


def _up_bwd(dout=P, dout_lo=None, dout_pitch=C + NB * 8, c_off=C, bin_ptr=P, bin_lo=None):
    lo = _ptrs(bin_lo) if dout_lo is not None else None
    return _lib.load().semseg_ppm_upsample_bwd(dout, dout_lo, dout_pitch, c_off, _ptrs(bin_ptr), lo, _bins(), NB,
                                               2, 9, 12, 8, None)


def _rs_fwd(x=P, x_lo=None, x_pitch=C, y=P, y_lo=None, y_pitch=C):
    return _lib.load().semseg_resize_bilinear_fwd(x, x_lo, x_pitch, 1, 59, 59, C, 30, 30, y, y_lo, y_pitch, None)


def _rs_bwd(dy=P, dy_lo=None, dy_pitch=C, dx=P, dx_lo=None, dx_pitch=C):
    return _lib.load().semseg_resize_bilinear_bwd(dy, dy_lo, dy_pitch, 1, 59, 59, C, 30, 30, dx, dx_lo, dx_pitch, None)


def _mp_fwd(x=P, x_lo=None, y=P, y_lo=None, argcode=P):
    return _lib.load().semseg_maxpool3x3s2_fwd(x, x_lo, y, y_lo, argcode, 1, 9, 9, C, None)


def _mp_bwd(argcode=P, dy=P, dy_lo=None, dx=P, dx_lo=None):
    return _lib.load().semseg_maxpool3x3s2_bwd(argcode, dy, dy_lo, dx, dx_lo, 1, 9, 9, C, None)


def _s2p(x=P, x_pitch=C, xp=P):
    return _lib.load().semseg_space_to_phases(x, x_pitch, 1, 9, 9, C, xp, None)


def _p2s(xp=P, x=P):
    return _lib.load().semseg_phases_to_space(xp, 1, 9, 9, C, x, None)


def _im2col(x=P, x_pitch=4, out=P):
    return _lib.load().semseg_im2col3x3s2(x, x_pitch, 1, 9, 9, 3, out, None)


def _rejected(call, name, what, **kw):
    lib = _lib.load()
    before = lib.semseg_launch_count()
    assert call(**kw) == -1, kw
    msg = lib.semseg_last_error()
    assert name.encode() in msg and what.encode() in msg, (kw, msg)
    assert lib.semseg_launch_count() == before, "a rejected call launched a kernel"


# (entry point, name in the message, its activation operands accessed with 16-byte vectors: (hi, lo, pitch or None))
CALLS = [
    (_pool, "ppm_pool", [("x", "x_lo", "x_pitch"), ("bin_ptr", "bin_lo", None)]),
    (_pool_bwd, "ppm_pool_bwd", [("dx", "dx_lo", "dx_pitch"), ("add", "add_lo", "add_pitch"),
                                 ("bin_ptr", "bin_lo", None)]),
    (_up, "ppm_upsample_concat", [("x", "x_lo", "x_pitch"), ("out", "out_lo", None), ("bin_ptr", "bin_lo", None)]),
    (_up_bwd, "ppm_upsample_bwd", [("dout", "dout_lo", None), ("bin_ptr", "bin_lo", None)]),
    (_rs_fwd, "resize_bilinear_fwd", [("x", "x_lo", "x_pitch"), ("y", "y_lo", "y_pitch")]),
    (_rs_bwd, "resize_bilinear_bwd", [("dy", "dy_lo", "dy_pitch"), ("dx", "dx_lo", "dx_pitch")]),
    (_mp_fwd, "maxpool3x3s2_fwd", [("x", "x_lo", None), ("y", "y_lo", None)]),
    (_mp_bwd, "maxpool3x3s2_bwd", [("dy", "dy_lo", None), ("dx", "dx_lo", None)]),
    (_s2p, "space_to_phases", [("x", None, "x_pitch"), ("xp", None, None)]),
    (_p2s, "phases_to_space", [("xp", None, None), ("x", None, None)]),
    (_im2col, "im2col3x3s2", [("out", None, None)]),
]
IDS = [c[1] for c in CALLS]


def _split(names):
    """Keyword arguments that make every activation operand of the call split (lo planes at an aligned address)."""
    return {lo: P for _, lo, _ in names if lo is not None}


@pytest.mark.parametrize("call,name,operands", CALLS, ids=IDS)
def test_misaligned_base_rejected_before_launch(call, name, operands):
    """Each operand in turn at a 2-byte and an 8-byte aligned base, plain and split; in split storage also the lo plane
    alone (a hi plane that is aligned does not make the lo plane aligned). The per-bin tables of ppm.cu are checked
    like the activations."""
    for hi, lo, _ in operands:
        for bad in (ODD, HALF):
            _rejected(call, name, "aligned", **{hi: bad})
            if lo is None:
                continue
            _rejected(call, name, "aligned", **dict(_split(operands), **{hi: bad}))
            _rejected(call, name, "aligned", **dict(_split(operands), **{lo: bad}))


@pytest.mark.parametrize("call,name,operands", [c for c in CALLS if any(p for _, _, p in c[2])],
                         ids=[c[1] for c in CALLS if any(p for _, _, p in c[2])])
def test_pitch_below_channels_rejected_before_launch(call, name, operands):
    """A pitch that is a multiple of 8 but smaller than C would make rows overlap (ppm_pool_bwd's dx_pitch was not
    checked at all; the rest checked only pitch % 8)."""
    for _, _, pitch in operands:
        if pitch is not None:
            _rejected(call, name, "pitch", **{pitch: C - 8})


def test_upsample_concat_output_narrower_than_the_concat_rejected():
    _rejected(_up, "ppm_upsample_concat", "bad args", out_pitch=C + NB * 8 - 8)


def test_upsample_bwd_slice_past_the_pitch_rejected():
    """dfeat_k reads channels c_off + k*Cr .. c_off + (k+1)*Cr of every dout pixel: a c_off that puts the last bin's
    slice past the pitch would read the next pixel's channels, and past the buffer at the last pixel."""
    width = C + NB * 8
    for c_off, pitch in ((C + 8, width), (width, width), (C, width - 8), (0, NB * 8 - 8)):
        _rejected(_up_bwd, "ppm_upsample_bwd", "exceed the pitch", c_off=c_off, dout_pitch=pitch)
    _rejected(_up_bwd, "ppm_upsample_bwd", "bad args", c_off=-8)


def test_maxpool_argcode_needs_8_byte_alignment():
    """argcode holds one byte per element, stored and loaded as one uint2 per 8 channels."""
    for bad in (ctypes.c_void_p(17), ctypes.c_void_p(20)):
        _rejected(_mp_fwd, "maxpool3x3s2_fwd", "8-byte aligned", argcode=bad)
        _rejected(_mp_bwd, "maxpool3x3s2_bwd", "8-byte aligned", argcode=bad)


def test_im2col_input_needs_8_byte_alignment():
    """im2col3x3s2 reads the (up to 3) input channels of a pixel as one uint2: an 8-byte aligned base (pitch 4) is
    accepted up to the next check, a 2- or 4-byte aligned one is not."""
    for bad in (ODD, ctypes.c_void_p(20)):
        _rejected(_im2col, "im2col3x3s2", "8-byte aligned", x=bad)
    # HALF (8-byte aligned) passes the input check and is stopped at the output (0x12, 16-byte uint4 stores)
    _rejected(_im2col, "im2col3x3s2", "0x12", x=HALF, out=ODD)


def test_slices_on_eight_channel_boundaries_pass_the_check():
    """What the network passes: ppm_pool_bwd's `add` as dout[..., :C] of the (C + nb*Cr)-wide concat gradient, split,
    lo plane behind the hi plane, and dx at pitch C. The call gets past the activation checks and is stopped by the
    next one (a bin table at 0x12), so nothing is launched."""
    m, width = 2 * 9 * 12, C + NB * 8
    plane = 2 * m * width                      # bytes per plane of the [M][width] bf16 concat gradient
    base = 1 << 20
    _rejected(_pool_bwd, "ppm_pool_bwd", "0x12", dx_lo=P, add=ctypes.c_void_p(base),
              add_lo=ctypes.c_void_p(base + plane), add_pitch=width, bin_ptr=ODD, bin_lo=P)
