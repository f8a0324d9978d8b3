"""CPU tier for frozen BatchNorm (eval-mode BN inside a network that trains): the one-pass backward kernel
(semseg_bn_bwd_frozen, csrc/bn.cu) rejects bad arguments with SEMSEG_E_INVALID before any CUDA call, and the oracle's
frozen-BN oracle (tests/frozen_oracle.py) without frozen layers is the oracle the reference goldens pin."""
import ctypes
import os

import numpy as np
import torch

from semseg_b200 import _lib
from tests import util
from tests.frozen_oracle import FrozenBNOracle, frozen_oracle_from

P = ctypes.c_void_p(16)      # never dereferenced: validation fails before any launch


def _err():
    return _lib.load().semseg_last_error()


def _call(dy=P, dy_lo=None, dy_pitch=64, y=P, y_lo=None, y_pitch=64, raw=P, raw_lo=None, raw_pitch=64, gamma=P,
          beta=P, rm=P, rv=P, eps=1e-5, M=100, C=64, relu=1, d_raw=P, d_raw_lo=None, d_raw_pitch=64, dres=P,
          dres_lo=None, dres_pitch=64, ws=P, ws_floats=1 << 30, sums=P):
    return _lib.load().semseg_bn_bwd_frozen(dy, dy_lo, dy_pitch, y, y_lo, y_pitch, raw, raw_lo, raw_pitch, gamma, beta,
                                            rm, rv, eps, M, C, relu, d_raw, d_raw_lo, d_raw_pitch, dres, dres_lo,
                                            dres_pitch, ws, ws_floats, sums, None)


def test_bn_bwd_frozen_validates_arguments():
    for kw in (dict(dy=None), dict(d_raw=None), dict(rm=None), dict(rv=None)):        # null required pointers
        assert _call(**kw) == -1, kw
        assert b"bn_bwd_frozen" in _err() and b"null" in _err()
    for kw in (dict(M=0), dict(M=-5), dict(C=0), dict(C=12), dict(C=-8)):            # M <= 0, C % 8 != 0
        assert _call(**kw) == -1, kw
        assert b"bn_bwd_frozen" in _err()
    assert _call(y=None, raw=None) == -1                                               # relu without a mask source
    assert b"relu" in _err()
    for kw in (dict(dy_pitch=56), dict(d_raw_pitch=56), dict(y_pitch=56), dict(raw_pitch=56), dict(dres_pitch=56),
               dict(dy_pitch=68), dict(d_raw_pitch=66)):                               # pitch < C, unaligned pitch
        assert _call(**kw) == -1, kw
        assert b"bn_bwd_frozen" in _err() and b"pitch" in _err()
    assert _call(ws=None) == -1 and b"workspace" in _err()                             # sums without workspace
    assert _call(ws_floats=100) == -1 and b"workspace" in _err()                       # workspace too small
    assert _call(dy_lo=P) == -1 and b"storage form" in _err()                          # split dy, plain d_raw
    assert _call(dy_lo=P, d_raw_lo=P, y_lo=P, raw_lo=P) == -1 and b"storage form" in _err()    # plain dres


def test_oracle_without_frozen_layers_reproduces_goldens(golden_dir):
    """FrozenBNOracle without frozen layers reproduces the training losses and running statistics of the reference goldens."""
    g = np.load(os.path.join(golden_dir, "pspnet50_65.npz"))
    torch.set_num_threads(8)
    model = util.build_pspnet(50, 150)
    orc, sd = frozen_oracle_from(model, "psp", frozen=(), layers=50, classes=150)
    x, y = util.synth(2, 65, 65, 150, seed=123)
    nbt = sd["layer4.2.bn3.num_batches_tracked"].clone()
    with torch.no_grad():
        _, main_loss, aux_loss = orc.train().forward(x, y)
    assert abs(main_loss.item() - float(g["main_loss"])) < 2e-5
    assert abs(aux_loss.item() - float(g["aux_loss"])) < 2e-5
    assert util.rel_l2(sd["layer4.2.bn3.running_mean"][:32], g["running_mean/layer4.2.bn3"]) < 1e-5
    assert int(sd["layer4.2.bn3.num_batches_tracked"]) == int(nbt) + 1


def test_oracle_frozen_layers_use_running_statistics():
    """A frozen name normalises with the running statistics and leaves them and num_batches_tracked untouched; the
    other layers of the same training network keep batch statistics."""
    from semseg_b200.resnet import Bottleneck
    torch.manual_seed(0)
    blk = Bottleneck(64, 16)
    for m in blk.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            torch.nn.init.uniform_(m.weight, 0.5, 1.5)
            torch.nn.init.normal_(m.bias, 0, 0.2)
            torch.nn.init.normal_(m.running_mean, 0, 0.3)
            torch.nn.init.uniform_(m.running_var, 0.5, 2.0)
    sd = {"layer1.0." + k: v.detach().clone() for k, v in blk.state_dict().items()}
    before = {k: v.clone() for k, v in sd.items()}
    orc = FrozenBNOracle(sd, frozen={"layer1.0.bn1", "layer1.0.bn3"}).train()
    x = torch.randn((2, 64, 9, 9))
    yo = orc.bottleneck(x, "layer1.0", 1, 1, False)
    # the same block through torch modules: bn1 / bn3 in eval mode, bn2 in training mode
    blk.train()
    blk.bn1.eval()
    blk.bn3.eval()
    t = torch.relu(blk.bn1(blk.conv1(x)))
    t = torch.relu(blk.bn2(torch.nn.functional.conv2d(t, blk.conv2.weight, padding=1)))
    ref = torch.relu(blk.bn3(blk.conv3(t)) + x)
    assert torch.allclose(yo, ref, rtol=1e-5, atol=1e-5)
    for name in ("bn1", "bn3"):
        for buf in ("running_mean", "running_var", "num_batches_tracked"):
            k = "layer1.0.%s.%s" % (name, buf)
            assert torch.equal(sd[k], before[k]), k
    assert not torch.equal(sd["layer1.0.bn2.running_mean"], before["layer1.0.bn2.running_mean"])
    assert int(sd["layer1.0.bn2.num_batches_tracked"]) == int(before["layer1.0.bn2.num_batches_tracked"]) + 1
