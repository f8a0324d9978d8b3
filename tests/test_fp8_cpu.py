"""CPU tier of FP8 (e4m3) inference (semseg_b200/fp8.py): the oracle's e4m3 rounding at hand-checked values, the stage
selection rule, every error of Fp8Eval that needs no GPU, and the argument checks of the new C entry points."""
import ctypes

import numpy as np
import pytest
import torch

from semseg_b200 import _lib
from semseg_b200.fp8 import Fp8Eval, fp8_stages
from semseg_b200.psanet import PSANet
from semseg_b200.pspnet import PSPNet
from tests import fp8_oracle as O


def _codes(vals):
    return O.e4m3(torch.tensor(vals, dtype=torch.float32)).view(torch.uint8).tolist()


def test_e4m3_rounding_hand_checked():
    # normals: 1 = 0x38, 1.125 = 0x39 (3 mantissa bits); ties to even between 1 and 1.125 and between 1.125 and 1.25
    assert _codes([1.0, 1.0625, 1.1875, 1.125, -1.0]) == [0x38, 0x38, 0x3A, 0x39, 0xB8]
    # largest finite 448 = 0x7E; 464 is the tie between 448 and (non-existent) 480: saturates to 448, as does 480 and inf
    assert _codes([448.0, 464.0, 480.0, 1e9, float("inf"), -480.0]) == [0x7E, 0x7E, 0x7E, 0x7E, 0x7E, 0xFE]
    # subnormals: 2^-9 = 0x01, 2^-10 is a tie between 0 and 2^-9 -> 0 (even), 3 * 2^-10 -> 2^-8 = 0x02
    assert _codes([2.0 ** -9, 2.0 ** -10, 3 * 2.0 ** -10, 7 * 2.0 ** -9, 2.0 ** -6]) == [0x01, 0x00, 0x02, 0x07, 0x08]
    assert _codes([0.0, -0.0]) == [0x00, 0x80]
    assert O.e4m3(torch.tensor([float("nan")])).float().isnan().all()


def test_quantize_and_pack_oracle():
    x = torch.tensor([1.0, -2.0, 100.0, 0.0], dtype=torch.bfloat16)
    qs, s = O.qscale_of(100.0)
    assert qs == np.float32(4.48) and s == np.float32(100.0) / np.float32(448.0)
    assert O.quantize(x, qs).float().tolist() == [4.5, -9.0, 448.0, 0.0]
    assert O.qscale_of(0.0) == (np.float32(1.0), np.float32(1.0))
    w = torch.randn(8, 16, 3, 3, generator=torch.Generator().manual_seed(0))
    w[3] = 0.0
    slab, sw = O.pack_weights(w)
    assert slab.shape == (9, 8, 16) and sw[3] == 1.0
    assert torch.equal(slab.view(torch.uint8)[4, 2], O.e4m3(w[2, :, 1, 1] * (448.0 / w[2].abs().max())).view(torch.uint8))
    deq = O.dequant_weights(w)
    assert float((deq - w.double()).abs().max() / w.abs().max()) < 2 ** -4


def _names(model):
    return [n for n, _, _ in fp8_stages(model)]


@pytest.mark.parametrize("layers", [50, 101])
def test_stage_selection_pspnet(layers):
    model = PSPNet(layers=layers, classes=19, pretrained=False).eval()
    names = _names(model)
    blocks = {50: (3, 4, 6, 3), 101: (3, 4, 23, 3)}[layers]
    # layer1: conv1 of every block and the downsample (Cin 128 / 256); conv2 / conv3 read 64 channels
    exp = ["layer1.0.conv1", "layer1.0.downsample.0"] + ["layer1.%d.conv1" % i for i in range(1, blocks[0])]
    for li in (2, 3, 4):
        for b in range(blocks[li - 1]):
            exp += ["layer%d.%d.%s" % (li, b, c) for c in ("conv1", "conv2", "conv3")]
            if b == 0:
                exp.append("layer%d.0.downsample.0" % li)
    exp += ["ppm.features.%d.1" % i for i in range(4)] + ["cls.0"]
    assert names == exp
    mods = dict(model.named_modules())
    assert all(mods[n].in_channels % 128 == 0 for n in names)
    assert "layer0.0" not in names and "cls.4" not in names and not any(n.startswith("aux") for n in names)


@pytest.mark.parametrize("psa_type,compact", [(0, False), (1, False), (2, False), (0, True), (2, True)])
def test_stage_selection_psanet(psa_type, compact):
    model = PSANet(layers=50, classes=19, psa_type=psa_type, compact=compact, pretrained=False).eval()
    names = _names(model)
    ctx = [n for n in names if n.startswith("psa")]
    exp = ["psa.reduce.0", "psa.attention.0"]
    if psa_type == 2:
        exp += ["psa.reduce_p.0", "psa.attention_p.0"]
    assert ctx == exp + ["psa.proj.0"]
    assert names[-1] == "cls.0" and "psa.attention.3" not in names


def test_fp8eval_rejects_what_it_cannot_run():
    model = PSPNet(layers=50, classes=5, pretrained=False)
    with pytest.raises(ValueError, match="CUDA only"):
        Fp8Eval(model.eval())
    with pytest.raises(TypeError, match="PSPNet or PSANet"):
        Fp8Eval(torch.nn.Conv2d(3, 3, 1))
    dp = torch.nn.DataParallel(model)
    dp.device_ids = [0, 1]           # what a two-GPU wrapper holds; no device is touched here
    with pytest.raises(ValueError, match="DataParallel over 2 devices"):
        Fp8Eval(dp)


def test_fp8eval_errors_before_any_launch(monkeypatch):
    """Training mode, running before freeze(), freeze() without calibration, a mismatched calibration, an input that
    needs a gradient, changed weights: clear errors, checked on the host before anything runs."""
    import semseg_b200.fp8 as fp8
    model = PSPNet(layers=50, classes=5, pretrained=False)
    monkeypatch.setattr(fp8, "_net_of", lambda m: m)          # a CPU model standing in for a CUDA one
    with pytest.raises(RuntimeError, match="training mode"):
        Fp8Eval(model.train())
    model.eval()
    q = Fp8Eval(model)
    with pytest.raises(RuntimeError, match="freeze"):
        q(torch.zeros(1, 3, 9, 9))
    with pytest.raises(RuntimeError, match="has not reached 51 FP8 stages"):
        q.freeze()
    cal = {n: 1.0 for n in _names(model)}
    bad = dict(cal)
    bad.pop("cls.0")
    bad["cls.4"] = 1.0
    with pytest.raises(ValueError, match="missing .*cls.0.*unknown .*cls.4"):
        Fp8Eval(model, calibration=bad)
    with pytest.raises(ValueError, match="finite"):
        Fp8Eval(model, calibration=dict(cal, **{"cls.0": float("nan")}))
    q = Fp8Eval(model, calibration=cal)
    assert q.calibration() == cal
    # freeze() stand-in: a plan whose stages carry the parameter keys of now
    stages = []
    for name, conv, bn in fp8_stages(model):
        st = fp8._Stage()
        st.name, st.conv, st.bn, st.key = name, conv, bn, fp8._param_key(conv, bn)
        stages.append(st)
    q._plan = fp8._Plan(stages)
    with pytest.raises(RuntimeError, match="does not require grad"):
        q._enter(torch.zeros(1, 3, 9, 9, requires_grad=True))
    q._enter(torch.zeros(1, 3, 9, 9))
    with torch.no_grad():
        model.layer3[1].conv2.weight.mul_(1.0)               # an optimizer-style in-place update bumps the version
    with pytest.raises(RuntimeError, match="layer3.1.conv2 changed since freeze"):
        q._enter(torch.zeros(1, 3, 9, 9))
    model.train()
    with pytest.raises(RuntimeError, match="training mode"):
        q._enter(torch.zeros(1, 3, 9, 9))


def test_calibration_round_trip_values():
    """calibration() -> Fp8Eval(calibration=...) keeps every fp32 amax bit for bit (device-free: the bits tensor lives
    wherever the model does)."""
    import semseg_b200.fp8 as fp8
    model = PSANet(layers=50, classes=5, psa_type=2, pretrained=False).eval()
    orig = fp8._net_of
    try:
        fp8._net_of = lambda m: m
        names = _names(model)
        rng = np.random.default_rng(0)
        cal = {n: float(np.float32(v)) for n, v in zip(names, rng.uniform(0.01, 300.0, len(names)))}
        cal[names[3]] = 0.0
        q = Fp8Eval(model, calibration=cal)
        assert q.calibration() == cal
        assert Fp8Eval(model, calibration=q.calibration()).calibration() == cal
    finally:
        fp8._net_of = orig


def test_entry_points_validate_before_any_cuda_call():
    lib = _lib.load()
    P = ctypes.c_void_p(256)
    err = lambda: lib.semseg_last_error()      # noqa: E731
    assert lib.semseg_fp8_quantize(P, 64, P, 64, 10, 60, 1.0, None) == -1 and b"C % 16" in err()
    assert lib.semseg_fp8_quantize(P, 72, P, 64, 10, 64, 1.0, None) == -1 and b"pitches" in err()
    assert lib.semseg_fp8_quantize(P, 64, P, 64, 10, 64, 0.0, None) == -1 and b"qscale" in err()
    assert lib.semseg_fp8_quantize(P, 64, P, 64, 10, 64, float("inf"), None) == -1 and b"qscale" in err()
    assert lib.semseg_fp8_quantize(ctypes.c_void_p(258), 64, P, 64, 10, 64, 1.0, None) == -1 and b"aligned" in err()
    assert lib.semseg_fp8_amax(P, 64, 10, 64, None, None) == -1 and b"fp8_amax" in err()
    assert lib.semseg_fp8_amax(P, 60, 10, 64, P, None) == -1 and b"pitch" in err()
    assert lib.semseg_fp8_pack_weights(P, 64, 24, 9, P, P, None) == -1 and b"Cin % 16" in err()
    assert lib.semseg_fp8_pack_weights(P, 64, 128, 10, P, P, None) == -1 and b"taps" in err()

    def desc(**kw):
        d = _lib.ConvDesc()
        d.N, d.H, d.W, d.Cin, d.Cout = 1, 8, 8, 256, 128
        d.x, d.Nin, d.Hin, d.Win, d.x_pitch = 256, 1, 8, 8, 256
        d.w, d.n_wtaps, d.w_rows, d.w_cols = 256, 1, 128, 256
        d.taps, d.img_mul = 1, 1
        d.epi_mode, d.y, d.y_pitch, d.e4m3 = 1, 256, 128, 1
        for k, v in kw.items():
            setattr(d, k, v)
        return d

    def fprop(**kw):
        return lib.semseg_conv_fprop(ctypes.byref(desc(**kw)), None)

    assert fprop(Cin=192, x_pitch=192, w_cols=192) == -1 and b"Cin % 128" in err()
    assert fprop(x_pitch=264) == -1 and b"x_pitch 264 must be a multiple of 16" in err()
    assert fprop(w_cols=264) == -1 and b"w_cols 264" in err()
    assert fprop(y8=256, y8_pitch=136, y8_qscale=1.0) == -1 and b"y8_pitch 136" in err()
    assert fprop(y8=256, y8_pitch=128, y8_qscale=0.0) == -1 and b"y8_qscale" in err()
    assert fprop(y8=256, y8_pitch=128, y8_qscale=float("nan")) == -1 and b"y8_qscale" in err()
    assert fprop(epi_mode=2) == -1 and b"AFFINE" in err()
    assert fprop(epi_mode=0) == -1 and b"AFFINE" in err()
    assert fprop(k_slices=2) == -1 and b"K-sliced" in err()
    assert fprop(stats_partial=256) == -1 and b"statistics" in err()
    assert fprop(x_lo=256) == -1 and b"split" in err()
    assert fprop(y=None) == -1 and b"without an output" in err()
    # the bf16 path refuses an e4m3 output
    assert fprop(e4m3=0, Cin=256, y8=256, y8_pitch=128, y8_qscale=1.0) == -1 and b"needs e4m3 operands" in err()


def test_freeze_rejects_non_finite_calibration(monkeypatch):
    """An infinite activation seen by calibrate() would give an infinite epilogue scale: freeze() refuses it."""
    import semseg_b200.fp8 as fp8
    model = PSPNet(layers=50, classes=5, pretrained=False).eval()
    monkeypatch.setattr(fp8, "_net_of", lambda m: m)
    q = Fp8Eval(model, calibration={n: 1.0 for n in _names(model)})
    q._bits[7] = int(np.array([np.inf], dtype=np.float32).view(np.int32)[0])
    with pytest.raises(RuntimeError, match="non-finite activations at 1 FP8 stages"):
        q.freeze()


def test_e4m3_mode_values_validated():
    lib = _lib.load()
    d = _lib.ConvDesc()
    d.N, d.H, d.W, d.Cin, d.Cout = 1, 8, 8, 256, 128
    d.x, d.Nin, d.Hin, d.Win, d.x_pitch = 256, 1, 8, 8, 256
    d.w, d.n_wtaps, d.w_rows, d.w_cols = 256, 1, 128, 256
    d.taps, d.img_mul, d.epi_mode, d.y, d.y_pitch, d.e4m3 = 1, 1, 1, 256, 128, 3
    assert lib.semseg_conv_fprop(ctypes.byref(d), None) == -1 and b"unpromoted" in lib.semseg_last_error()
