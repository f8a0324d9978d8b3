"""CPU tier of PSANet's compact and softmax-free attention:
  * the fp32 oracle reproduces the reference's own compact / psa_softmax=False PSANet50 (tests/golden/psanet50_65_*.npz,
    written by tests/golden/make_psa_variants_golden.py) to the tolerances of test_oracle_cpu.py;
  * semseg_psa_attend_ex / semseg_psa_attend_bwd_attn_ex reject bad form bits, geometries and NULL operands before any
    CUDA call;
  * functional.psa_attend_supported: which geometries the fused kernels take, in the window and the compact form."""
import ctypes
import os

import numpy as np
import pytest
import torch

from semseg_b200 import _lib
from tests import util

VARIANTS = {  # fixture tag -> (psa_type, compact, psa_softmax, mask)
    "psanet50_65_t2_compact": (2, True, True, 5),
    "psanet50_65_t2_nosoftmax": (2, False, False, 9),
    "psanet50_65_t1_compact_nosoftmax": (1, True, False, 5),
    "psanet50_65_t0_compact": (0, True, True, 5),
}


def build_variant(psa_type, compact, softmax, mask):
    from semseg_b200.psanet import PSANet
    torch.manual_seed(0)
    return PSANet(layers=50, classes=150, zoom_factor=8, dropout=0.0, psa_type=psa_type, compact=compact,
                  shrink_factor=2, mask_h=mask, mask_w=mask, normalization_factor=1.0, psa_softmax=softmax,
                  pretrained=False)


@pytest.mark.parametrize("tag", sorted(VARIANTS))
def test_oracle_matches_reference_psa_variant(tag, golden_dir):
    psa_type, compact, softmax, mask = VARIANTS[tag]
    g = np.load(os.path.join(golden_dir, tag + ".npz"))
    torch.set_num_threads(8)
    model = build_variant(psa_type, compact, softmax, mask)
    sdm = model.state_dict()
    wkeys = [k for k in g.files if k.startswith("wsum/")]
    assert len(wkeys) >= 5
    for k in wkeys:                       # identical construction order => identical seeded weights as the reference
        a, s = g[k]
        name = k[len("wsum/"):]
        assert abs(float(sdm[name].double().abs().sum()) - a) <= 1e-9 * max(1.0, abs(a)), name
        assert abs(float(sdm[name].double().sum()) - s) <= 1e-6 * max(1.0, abs(a)), name
    orc, sd = util.oracle_from(model, "psa", layers=50, classes=150, psa_type=psa_type, compact=compact,
                               mask_h=mask, mask_w=mask, psa_softmax=softmax)
    x, y = util.synth(2, 65, 65, 150, seed=321)
    orc.train()
    out, main_loss, aux_loss = orc.forward(x, y)
    (main_loss + 0.4 * aux_loss).backward()
    assert abs(main_loss.item() - float(g["main_loss"])) < 2e-5
    assert abs(aux_loss.item() - float(g["aux_loss"])) < 2e-5
    assert (out.numpy().astype(np.int16) != g["argmax"]).mean() < 2e-3
    for k in g.files:
        if k.startswith("gradnorm/"):
            name = k[len("gradnorm/"):]
            got = sd[name].grad.double().norm().item()
            assert abs(got - float(g[k])) <= 2e-3 * float(g[k]) + 1e-9, (name, got, float(g[k]))
    tot = float(torch.sqrt(sum((v.grad.double() ** 2).sum() for v in sd.values() if v.grad is not None)))
    assert abs(tot - float(g["gradnorm_total"])) <= 1e-3 * float(g["gradnorm_total"])
    orc.eval()
    with torch.no_grad():
        logits = orc.forward(x)
    assert util.rel_l2(logits[:, :, ::8, ::8], g["eval_logits_s8"]) < 1e-4
    assert util.rel_l2(sd["layer4.2.bn3.running_mean"][:32], g["running_mean/layer4.2.bn3"]) < 1e-5


DENSE, NOSM = _lib.PSA_DENSE, _lib.PSA_NO_SOFTMAX


def _attend(form, stats=True, a_pitch=9, H=3, W=3, mH=3, mW=3, C=512, pitch=512):
    # semseg_psa_attend_ex(mode, psa_type, form, attn, a_pitch, feat, feat_lo, feat_pitch, stats, out, out_lo, out_pitch,
    #                      N, H, W, mH, mW, C, scale, stream)
    P = ctypes.c_void_p(16)
    return _lib.load().semseg_psa_attend_ex(0, 0, form, P, a_pitch, P, None, pitch, P if stats else None, P, None, pitch,
                                            1, H, W, mH, mW, C, 1.0, None)


def _attn_grad(form, stats=True, out=True, a_pitch=9, H=3, W=3, mH=3, mW=3, C=512, pitch=512):
    # semseg_psa_attend_bwd_attn_ex(psa_type, form, attn, a_pitch, stats, feat, feat_lo, feat_pitch, out, out_lo, out_pitch,
    #                               dout, dout_lo, dout_pitch, dattn, N, H, W, mH, mW, C, scale, stream)
    P = ctypes.c_void_p(16)
    return _lib.load().semseg_psa_attend_bwd_attn_ex(1, form, P, a_pitch, P if stats else None, P, None, pitch,
                                                     P if out else None, None, pitch, P, None, pitch, P, 1, H, W, mH, mW,
                                                     C, 1.0, None)


def _rejects(status, *words):
    msg = _lib.load().semseg_last_error()
    assert status == -1 and all(w.encode() in msg for w in words), msg


def test_psa_attend_ex_validates_before_any_cuda_call():
    for call, fn in ((_attend, "psa_attend"), (_attn_grad, "psa_attend_bwd_attn")):
        _rejects(call(4), fn, "unknown form bits")
        _rejects(call(-1), fn, "unknown form bits")
        # dense form: mH*mW == H*W and a_pitch >= H*W, no parity condition
        _rejects(call(DENSE, H=3, W=4, mH=3, mW=3, a_pitch=12), fn, "mask geometry", "dense")
        _rejects(call(DENSE | NOSM, H=3, W=4, mH=2, mW=6, a_pitch=11), fn, "mask geometry")
        # an even dense mask passes the geometry check and is stopped by the next one (feature width / bad pitch)
        _rejects(call(DENSE, H=4, W=4, mH=4, mW=4, a_pitch=16, C=256, pitch=250), fn)
        assert b"mask geometry" not in _lib.load().semseg_last_error()
        # window form keeps the odd-mask checks, with and without softmax
        _rejects(call(NOSM, H=4, W=4, mH=4, mW=4, a_pitch=16), fn, "mask geometry")
        _rejects(call(0, H=4, W=4, mH=3, mW=3, a_pitch=8), fn, "mask geometry")
        # stats may be NULL only without softmax
        _rejects(call(0, stats=False), fn, "stats are required")
        _rejects(call(DENSE, stats=False, H=3, W=3, mH=3, mW=3), fn, "stats are required")
        _rejects(call(NOSM, stats=False, C=256, pitch=250), fn)
        assert b"stats" not in _lib.load().semseg_last_error()
        # W <= 128 stays, in the dense form too
        _rejects(call(DENSE, H=1, W=200, mH=1, mW=200, a_pitch=200), fn, "128")
    # C == 512 in the forward, C % 64 == 0 in the logit gradient
    _rejects(_attend(DENSE | NOSM, C=256, pitch=256), "feature width must be 512")
    _rejects(_attn_grad(DENSE | NOSM, C=100, pitch=104), "C % 64 == 0")
    # out may be NULL in the logit gradient only without softmax
    _rejects(_attn_grad(0, out=False), "psa_attend_bwd_attn", "out is required")
    _rejects(_attn_grad(DENSE, out=False), "out is required")
    _rejects(_attn_grad(NOSM, out=False, pitch=250), "bad pitch")
    _rejects(_attn_grad(DENSE | NOSM, stats=False, out=False, pitch=250), "bad pitch")


def test_psa_attend_supported_decisions():
    from semseg_b200.functional import psa_attend_supported as ok

    def feat(h, w, c=512):
        return torch.empty((2, h, w, c), dtype=torch.bfloat16)
    # window form: odd masks of any size, 512 channels, at most 128 columns
    assert ok(feat(5, 5), 9, 9) and ok(feat(30, 30), 59, 59) and ok(feat(5, 5), 5, 5) and ok(feat(9, 12), 9, 7)
    assert not ok(feat(5, 5), 8, 9) and not ok(feat(5, 5), 9, 4)
    assert not ok(feat(5, 130), 9, 9) and not ok(feat(5, 5, 256), 9, 9)
    # compact (dense) form: exactly h*w mask entries, whatever their parity
    assert ok(feat(5, 5), 5, 5, compact=True) and ok(feat(30, 30), 30, 30, compact=True)
    assert ok(feat(4, 6), 4, 6, compact=True) and ok(feat(4, 6), 3, 8, compact=True)
    assert not ok(feat(5, 5), 9, 9, compact=True) and not ok(feat(5, 5), 5, 4, compact=True)
    assert not ok(feat(1, 130), 1, 130, compact=True) and not ok(feat(5, 5, 256), 5, 5, compact=True)
    # the split storage form [2, N, h, w, C] is judged on the same trailing dimensions
    assert ok(torch.empty((2, 2, 5, 5, 512), dtype=torch.bfloat16), 5, 5, compact=True)
