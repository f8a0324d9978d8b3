"""CPU tier for input gradients (csrc/layout.cu stem dgrad, semseg_b200/functional.py): the stem dgrad entry point rejects
bad arguments with SEMSEG_E_INVALID and a message before any CUDA call; `_bn_mode` takes each row of the behaviour
contract (INTEGRATION.md §4); the fp32 oracle's own input-gradient floor lies below the GPU tier's tolerance."""
import ctypes

import pytest
import torch
import torch.nn as nn

from semseg_b200 import _lib
from semseg_b200 import functional as SF
from tests import input_grad_floor

P = ctypes.c_void_p(16)      # never dereferenced: validation fails before any launch


def _err():
    return _lib.load().semseg_last_error()


def _call(dy=P, dy_lo=None, pitch=64, N=2, Ho=None, Wo=None, H=65, W=64, Cin=3, Cout=64, wp=P, split=0, dx=P):
    Ho = (H - 1) // 2 + 1 if Ho is None else Ho
    Wo = (W - 1) // 2 + 1 if Wo is None else Wo
    return _lib.load().semseg_stem_dgrad3x3s2(dy, dy_lo, pitch, N, Ho, Wo, H, W, Cin, Cout, wp, split, dx, None)


def test_stem_dgrad_validates_arguments():
    for kw in ("dy", "wp", "dx"):
        assert _call(**{kw: None}) == -1 and b"stem_dgrad3x3s2" in _err() and b"null" in _err(), kw
    for cin in (0, 4, 8):
        assert _call(Cin=cin) == -1 and b"stem_dgrad3x3s2" in _err() and (b"Cin=%d" % cin) in _err()
    for cout in (32, 128):
        assert _call(Cout=cout, pitch=128) == -1 and (b"Cout=64 (got %d)" % cout) in _err()
    assert _call(Ho=34) == -1 and b"Ho=(H-1)/2+1" in _err()              # 65 rows -> 33 conv-output rows
    assert _call(Wo=33) == -1 and b"Wo=(W-1)/2+1" in _err()              # 64 columns -> 32
    assert _call(N=0) == -1 and b"stem_dgrad3x3s2" in _err()
    assert _call(H=0, Ho=0) == -1
    assert _call(pitch=60) == -1 and b"pitch" in _err()                  # pitch < Cout
    assert _call(pitch=68) == -1 and b"pitch" in _err()                  # not a multiple of 8
    assert _call(dy_lo=P, split=0) == -1 and b"dy_lo" in _err()          # a lo plane without a split slab
    assert _call(dy_lo=None, split=1) == -1 and b"dy_lo" in _err()       # a split slab without the lo plane
    assert _call(dy_lo=P, split=2) == -1 and b"wp_split" in _err()
    assert _call(dy=ctypes.c_void_p(24)) == -1 and b"aligned" in _err()


def _bn(training_bn=False):
    bn = nn.BatchNorm2d(8)
    bn.train(training_bn)
    return bn


def _t(grad):
    return torch.zeros(2, requires_grad=grad)


@pytest.mark.parametrize("net_training, x_grad, params_grad, want", [
    (True, False, True, "frozen"),       # training with frozen BN: as before
    (True, True, True, "frozen"),
    (True, True, False, "frozen"),       # adversarial training of a frozen-BN network
    (True, False, False, "eval"),        # nothing needs a gradient
    (False, False, True, "eval"),        # validate(): eval network, input without gradient -> detached single kernel
    (False, True, False, "frozen"),      # attack: eval network, frozen parameters, x.requires_grad
    (False, True, True, "frozen"),       # eval network, parameters and input need gradients
    (False, False, False, "eval"),
], ids=["train-params", "train-x-params", "train-x", "train-none", "validate", "eval-attack", "eval-x-params",
        "eval-none"])
def test_bn_mode_contract(net_training, x_grad, params_grad, want):
    bn = _bn()
    x, w = _t(x_grad), _t(params_grad)
    with SF.network_mode(net_training):
        assert SF._bn_mode(bn, (x, None), (w, w, w)) == want
        with torch.no_grad():                                    # grad disabled: always the detached single kernel
            assert SF._bn_mode(bn, (x, None), (w, w, w)) == "eval"
        assert SF._bn_mode(_bn(True), (x, None), (w,)) == "batch"    # BN in training mode: batch statistics
        # the residual counts as an activation input, never as a parameter
        assert SF._bn_mode(bn, (_t(False), _t(True)), (_t(False),)) == "frozen"


def test_bn_mode_eval_network_whose_input_needs_no_grad_stays_detached():
    """validate() on PSANet: the attention conv's fp32 logits keep a backward to its weight, so the activations after the
    attention need a gradient although the network's input does not. The eval network stays on the detached path; with
    an input that needs a gradient the same stage is differentiable."""
    bn, act, w = _bn(), _t(True), _t(True)
    with SF.network_mode(False, input_grad=False):
        assert SF._bn_mode(bn, (act, None), (w,)) == "eval"
    with SF.network_mode(False, input_grad=True):
        assert SF._bn_mode(bn, (act, None), (w,)) == "frozen"
    with SF.network_mode(True, input_grad=False):               # a training network: as before
        assert SF._bn_mode(bn, (act, None), (w,)) == "frozen"


class _Probe(torch.nn.Module):
    @SF.network_forward
    def forward(self, x):
        return SF._net.training, SF._net.input_grad


def test_network_forward_records_whether_the_input_needs_grad():
    m = _Probe()
    assert m(_t(True)) == (True, True) and m(_t(False)) == (True, False)
    assert m.eval()(x=_t(True)) == (False, True)


def test_bn_mode_eval_network_ignores_parameters():
    """The reference's validate() passes an input that needs no gradient while every parameter requires one: the eval
    network stays on the detached path, stage by stage and in the fused Bottleneck decision alike."""
    from semseg_b200.resnet import Bottleneck
    blk = Bottleneck(64, 16, downsample=nn.Sequential(nn.Conv2d(64, 64, 1, bias=False), nn.BatchNorm2d(64))).eval()
    x = _t(False)
    params = [p for p in blk.parameters()]
    assert all(p.requires_grad for p in params)
    with SF.network_mode(False):
        assert {SF._bn_mode(b, (x,), params) for b in (blk.bn1, blk.bn2, blk.bn3, blk.downsample[1])} == {"eval"}
        assert {SF._bn_mode(b, (_t(True),), params) for b in (blk.bn1, blk.bn2)} == {"frozen"}


def test_oracle_input_grad_floor_below_tolerance():
    """The fp32 oracle's x.grad against itself (PSPNet50 65x65, eval, frozen parameters): 1e-6 input perturbation and
    float64 leave it to ~1e-6; a perturbation at bf16x3's operand scale (2^-17) flips ReLU masks and moves it by ~1e-2.
    The GPU tier's bf16x3 bound is three times that floor."""
    torch.manual_seed(0)
    tiny, op_scale, f64 = input_grad_floor.measure_floor()
    assert tiny < 1e-4 and f64 < 1e-4, (tiny, f64)
    assert op_scale <= input_grad_floor.INPUT_GRAD_TOL / 2, op_scale
