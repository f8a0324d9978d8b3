"""CPU tier for the RMI (+ BCE + cross-entropy) loss on the fused tail (csrc/tail.cu RMI kernels): the float64 contract
of the GPU tests agrees with a second, literal statement of the paper's code on loss and gradient, its closed-form
gradient passes gradcheck, RMILoss validates its options, `fused_tail_supported` takes the native tail exactly for an
RMILoss of this type, and the new entry points reject bad arguments with SEMSEG_E_INVALID and a message before any
CUDA call."""
import ctypes
import math

import pytest
import torch
import torch.nn as nn

from semseg_b200 import _lib
from semseg_b200 import functional as SF
from semseg_b200.losses import DiceLoss, RMILoss
from tests.rmi_oracle import rmi_contract, rmi_grad, rmi_literal

P = ctypes.c_void_p(16)      # never dereferenced: validation fails before any launch


def _err():
    return _lib.load().semseg_last_error()


def _case(seed, n=2, c=5, h=22, w=19, p_ignore=0.1, absent=True):
    """float64 logits [N,C,H,W] and a target with ignored and out-of-range labels and (absent) class c - 1 missing."""
    g = torch.Generator().manual_seed(seed)
    z = torch.randn((n, c, h, w), generator=g, dtype=torch.float64) * 2
    # blocky targets, so the pooled one-hot maps vary between cells
    t = torch.randint(0, c - 1 if absent else c, (n, (h + 2) // 3, (w + 2) // 3), generator=g)
    t = t.repeat_interleave(3, 1).repeat_interleave(3, 2)[:, :h, :w].contiguous()
    t[torch.rand((n, h, w), generator=g) < p_ignore] = 255
    t[torch.rand((n, h, w), generator=g) < 0.03] = c + 3
    t[torch.rand((n, h, w), generator=g) < 0.03] = -2
    return z, t


def _literal_grad(z, t, **kw):
    x = z.clone().requires_grad_(True)
    loss = rmi_literal(x, t, **kw)
    (g,) = torch.autograd.grad(loss, x)
    return loss.detach(), g


# ------------------------------------------------------------------------------------------------ oracle
CASES = [
    dict(seed=0),                                   # H, W not multiples of 4, ignore / out-of-range, absent class
    dict(seed=1, h=12, w=12),                       # the minimum: one neighbourhood (K = 1)
    dict(seed=2, h=16, w=27, c=3, absent=False),    # every class present
    dict(seed=3, n=1, h=13, w=18, c=4, p_ignore=0.5),
]


@pytest.mark.parametrize("ce_weight", [0.0, 1.0])
@pytest.mark.parametrize("bce_weight", [0.0, 0.5, 1.0])
@pytest.mark.parametrize("case", range(len(CASES)))
def test_contract_agrees_with_literal_statement(case, bce_weight, ce_weight):
    z, t = _case(**CASES[case])
    kw = dict(bce_weight=bce_weight, alpha=5e-4, ce_weight=ce_weight)
    res = rmi_contract(z, t, **kw)
    lit, glit = _literal_grad(z, t, **kw)
    assert abs(float(res["loss"]) - float(lit)) <= 1e-10 * max(1.0, abs(float(lit)))
    g = rmi_grad(z, t, **kw, res=res)
    assert float((g - glit).abs().max()) <= 1e-9 * max(float(glit.abs().max()), 1e-12)


def test_contract_hand_values():
    z, t = _case(5, n=2, c=4, h=20, w=17)
    res = rmi_contract(z, t, bce_weight=0.25, alpha=1e-3, ce_weight=0.5)
    assert res["Y"].shape == (2, 4, 5, 4) and res["K"] == 3 * 2
    # bce / (n_valid + 1), with n_valid the valid pixel count over the whole call
    valid = (t != 255) & (t >= 0) & (t < 4)
    assert res["nv"] == int(valid.sum())
    loss = 0.25 * res["bce"] + 0.75 * res["r"].sum() / 18 + 0.5 * res["ce"]
    assert abs(float(loss) - float(res["loss"])) < 1e-12
    # an absent class (c = 3): S_ab = 0, so r is that of the prediction-free posterior and its dr/dQ is 0
    assert float(res["dQ"][:, 3].abs().max()) == 0.0


def test_nothing_valid():
    z, _ = _case(6, c=3, h=14, w=15)
    t = torch.full((2, 14, 15), 255, dtype=torch.int64)
    t[0, 0, 0] = 7                                    # out of range: not valid either
    for bw in (0.0, 0.5):
        res = rmi_contract(z, t, bce_weight=bw, alpha=5e-4, ce_weight=1.0)
        assert res["nv"] == 0 and float(res["bce"]) == 0.0 and float(res["ce"]) == 0.0
        assert torch.allclose(res["r"], torch.full_like(res["r"], 4.5 * math.log(5e-4)), rtol=0, atol=1e-12)
        assert float(rmi_grad(z, t, bce_weight=bw, ce_weight=1.0).abs().max()) == 0.0
        lit, glit = _literal_grad(z, t, bce_weight=bw, ce_weight=1.0)
        assert abs(float(lit) - float(res["loss"])) < 1e-12 and float(glit.abs().max()) == 0.0


def test_pixels_outside_the_pooled_rows_reach_bce_only():
    z, t = _case(7, n=1, c=3, h=19, w=17, p_ignore=0.0)
    g = rmi_grad(z, t, bce_weight=0.0, ce_weight=0.0)
    assert float(g[..., 16:, :].abs().max()) == 0.0 and float(g[..., :, 16:].abs().max()) == 0.0
    assert float(g[..., :16, :16].abs().max()) > 0.0
    g = rmi_grad(z, t, bce_weight=0.5, ce_weight=0.0)
    valid = (t >= 0) & (t < 3)
    assert torch.equal(g[..., 16:, :].abs().amax(1) > 0, valid[:, 16:, :])


class _Closed(torch.autograd.Function):
    @staticmethod
    def forward(ctx, z, t, bw, cw):
        ctx.save_for_backward(z, t)
        ctx.bw, ctx.cw = bw, cw
        return rmi_contract(z, t, bce_weight=bw, ce_weight=cw)["loss"]

    @staticmethod
    def backward(ctx, g):
        z, t = ctx.saved_tensors
        return g * rmi_grad(z, t, bce_weight=ctx.bw, ce_weight=ctx.cw), None, None, None


@pytest.mark.parametrize("bw,cw", [(0.0, 0.0), (0.5, 1.0)])
def test_closed_form_gradcheck(bw, cw):
    z, t = _case(8, n=1, c=3, h=13, w=14)
    z = (z * 0.5).requires_grad_(True)
    assert torch.autograd.gradcheck(lambda x: _Closed.apply(x, t, bw, cw), (z,), eps=1e-6, atol=1e-7, rtol=1e-4)


# ------------------------------------------------------------------------------------------------ RMILoss module
def test_rmi_loss_validation():
    d = RMILoss()
    assert (d.ignore_index, d.bce_weight, d.pos_alpha, d.ce_weight) == (255, 0.5, 5e-4, 0.0)
    d = RMILoss(ignore_index=-1, bce_weight=1, pos_alpha=1, ce_weight=2)
    assert (d.ignore_index, d.bce_weight, d.pos_alpha, d.ce_weight) == (-1, 1.0, 1.0, 2.0)
    assert isinstance(d.bce_weight, float) and "pos_alpha=1" in repr(d) and "ce_weight=2" in repr(d)
    assert list(d.state_dict()) == []
    for kw in ({"ignore_index": 255.0}, {"ignore_index": True}, {"bce_weight": "1"}, {"pos_alpha": None},
               {"ce_weight": True}, {"bce_weight": torch.tensor(0.5)}):
        with pytest.raises(TypeError):
            RMILoss(**kw)
    for kw in ({"bce_weight": -0.1}, {"bce_weight": 1.01}, {"bce_weight": float("nan")}, {"pos_alpha": 0.0},
               {"pos_alpha": -1e-4}, {"pos_alpha": float("inf")}, {"ce_weight": -1.0}, {"ce_weight": float("nan")}):
        with pytest.raises(ValueError):
            RMILoss(**kw)


def test_rmi_loss_has_no_cpu_fallback():
    crit = RMILoss(ce_weight=1.0)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        crit(torch.zeros((1, 3, 12, 12)), torch.zeros((1, 12, 12), dtype=torch.int64))
    with pytest.raises(ValueError, match="256 classes"):
        crit(torch.zeros((1, 257, 12, 12)), torch.zeros((1, 12, 12), dtype=torch.int64))
    with pytest.raises(ValueError, match="expected"):
        crit(torch.zeros((1, 3, 12, 12)), torch.zeros((1, 12, 11), dtype=torch.int64))
    for h, w in ((11, 12), (12, 11), (5, 40)):
        with pytest.raises(ValueError, match="at least 12"):
            crit(torch.zeros((1, 3, h, w)), torch.zeros((1, h, w), dtype=torch.int64))


# ------------------------------------------------------------------------------------------------ fused_tail_supported
class _SubclassRMI(RMILoss):
    pass


def _target(n, h, w):
    return torch.zeros((n, h, w), dtype=torch.int64)


@pytest.mark.parametrize("zoom", [1, 2, 4, 8])
def test_fused_tail_decisions(zoom):
    x_size = torch.Size((2, 3, 97, 113))                    # -> 13 x 15 logits
    logits = torch.zeros((2, 13, 15, 21))
    ho, wo = zoom * 12 + 1, zoom * 14 + 1
    y = _target(2, ho, wo)
    for crit in (RMILoss(), RMILoss(bce_weight=0.0, pos_alpha=1e-3, ce_weight=1.0)):
        assert SF.fused_tail_supported(crit, None, y, zoom, x_size)
        assert SF.fused_tail_supported(crit, logits, y, zoom)
        assert SF.fused_tail_supported(crit, torch.zeros((2, 13, 15, 256)), y, zoom)
        assert not SF.fused_tail_supported(crit, torch.zeros((2, 13, 15, 257)), y, zoom)
        for other in {1, 2, 4, 8} - {zoom}:
            yo = _target(2, other * 12 + 1, other * 14 + 1)
            assert not SF.fused_tail_supported(crit, logits, yo, zoom)
        assert not SF.fused_tail_supported(crit, logits, y.int(), zoom)
        assert not SF.fused_tail_supported(crit, logits, y[0], zoom)
        assert not SF.fused_tail_supported(crit, logits, y, 3)
    assert not SF.fused_tail_supported(_SubclassRMI(), None, y, zoom, x_size)
    assert not SF.fused_tail_supported(_SubclassRMI(), logits, y, zoom)
    for crit in (nn.CrossEntropyLoss(ignore_index=255), DiceLoss()):
        assert SF.fused_tail_supported(crit, logits, y, zoom)


def test_fused_tail_rmi_minimum_size():
    """12 x 12 is the smallest target (three pooled cells each way); smaller ones keep the ATen tail."""
    for zoom in (1, 2, 4, 8):
        for h, w in ((12, 12), (12, 40), (40, 12), (11, 40), (40, 11)):
            hl, wl = (h - 1) // zoom + 1, (w - 1) // zoom + 1
            ho, wo = zoom * (hl - 1) + 1, zoom * (wl - 1) + 1
            ok = ho >= 12 and wo >= 12
            assert SF.fused_tail_supported(RMILoss(), torch.zeros((1, hl, wl, 5)), _target(1, ho, wo), zoom) == ok
            assert SF.fused_tail_supported(nn.CrossEntropyLoss(), torch.zeros((1, hl, wl, 5)), _target(1, ho, wo),
                                           zoom)


def test_fused_tail_rmi_width_limit():
    """The RMI rows kernel stages 8 bytes per pixel of Z rows in 224 KB: 3584 columns at zoom 8, 28672 at zoom 1."""
    for zoom, limit in ((8, 3584), (4, 7168), (2, 14336), (1, 28672)):
        for want, ok in ((limit, True), (limit + zoom, False)):
            w = (want - 1) // zoom + 1
            wo = zoom * (w - 1) + 1
            assert (wo <= limit) == ok
            logits = torch.zeros((1, 13, w, 19))
            y = _target(1, zoom * 12 + 1, wo)
            assert SF.fused_tail_supported(RMILoss(), logits, y, zoom) == ok, (zoom, wo)


# ------------------------------------------------------------------------------------------------ C-ABI validation
def _rfwd(logits=P, pitch=21, N=2, h=9, w=7, C=21, target=P, Ho=None, Wo=None, zoom=4, bce_weight=0.5,
          pos_alpha=5e-4, ce_weight=1.0, ws=P, loss=P, amax=P, lse=P, pooled=P, table=P):
    Ho = zoom * (h - 1) + 1 if Ho is None else Ho
    Wo = zoom * (w - 1) + 1 if Wo is None else Wo
    return _lib.load().semseg_upsample_ce_rmi_fwd(logits, pitch, N, h, w, C, target, Ho, Wo, zoom, 255, bce_weight,
                                                  pos_alpha, ce_weight, ws, loss, amax, lse, pooled, table, None)


def _rbwd(logits=P, pitch=21, N=2, h=9, w=7, C=21, target=P, Ho=None, Wo=None, zoom=4, lse=P, pooled=P, table=P,
          g=P, ws=P, dl=P):
    Ho = zoom * (h - 1) + 1 if Ho is None else Ho
    Wo = zoom * (w - 1) + 1 if Wo is None else Wo
    return _lib.load().semseg_upsample_ce_rmi_bwd(logits, pitch, N, h, w, C, target, Ho, Wo, zoom, 255, lse, pooled,
                                                  table, g, ws, dl, None)


@pytest.mark.parametrize("call", [_rfwd, _rbwd], ids=["fwd", "bwd"])
def test_rmi_entry_points_validate_shapes(call):
    assert call(zoom=3, Ho=25, Wo=19) == -1 and b"zoom 3" in _err()
    for zoom in (1, 2, 4, 8):
        assert call(zoom=zoom, Ho=zoom * 8 + 2) == -1 and (b"Ho=%d(h-1)+1" % zoom) in _err()
    assert call(logits=None) == -1 and b"null" in _err()
    assert call(target=None) == -1 and b"null" in _err()
    assert call(C=257, pitch=257) == -1 and b"C<=256" in _err()
    assert call(pitch=20) == -1 and b"upsample_ce" in _err()
    assert call(N=0) == -1 and b"bad sizes" in _err()
    # too small a target: fewer than 3 pooled cells in a direction
    assert call(zoom=1, h=11, w=40) == -1 and b"12x12" in _err()
    assert call(zoom=2, h=20, w=6) == -1 and b"12x12" in _err()
    # 8-byte staged words: at most 3584 output columns at zoom 8
    assert call(zoom=8, w=450) == -1 and b"too large" in _err() and b"at most 3584" in _err()
    assert call(zoom=1, h=12, w=28673) == -1 and b"too large" in _err()


def test_rmi_entry_points_validate_options_and_outputs():
    for kw, bads in (("bce_weight", (-0.01, 1.01, float("nan"))), ("pos_alpha", (0.0, -1.0, float("nan"),
                                                                                   float("inf"))),
                     ("ce_weight", (-0.01, float("nan"), float("inf")))):
        for bad in bads:
            assert _rfwd(**{kw: bad}) == -1 and kw.encode() in _err(), (kw, bad)
    for kw in ("ws", "loss", "lse", "pooled", "table"):
        assert _rfwd(**{kw: None}) == -1 and b"upsample_ce_rmi_fwd" in _err() and b"null" in _err(), kw
    assert _rfwd(ws=ctypes.c_void_p(20)) == -1 and b"aligned" in _err()
    assert _rfwd(pooled=ctypes.c_void_p(18)) == -1 and b"aligned" in _err()
    assert _rfwd(table=ctypes.c_void_p(17)) == -1 and b"aligned" in _err()
    for kw in ("lse", "pooled", "table", "g", "ws", "dl"):
        assert _rbwd(**{kw: None}) == -1 and b"upsample_ce_rmi_bwd" in _err() and b"null" in _err(), kw
    assert _rbwd(table=ctypes.c_void_p(18)) == -1 and b"aligned" in _err()


def test_rmi_workspace_sizes():
    lib = _lib.load()
    for zoom in (1, 2, 4, 8):
        n, h, w, c = 2, 60, 61, 150
        ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
        ctas = n * h * ((wo + 127) // 128)
        rows, cols = max(zoom, 4), {1: 32, 2: 64, 4: 128, 8: 128}[zoom]
        pool_ctas = n * -(-ho // rows) * -(-wo // cols)
        assert (lib.semseg_upsample_ce_rmi_workspace_floats(n, ho, wo, c, zoom) ==
                2 * n * c * 190 + 2 * ctas + pool_ctas)
        assert (lib.semseg_upsample_ce_rmi_bwd_workspace_floats(n, ho, wo, w, c, zoom) ==
                lib.semseg_upsample_ce_zoom_bwd_workspace_floats(n, ho, w, c, zoom) + n * c * (ho // 4) * (wo // 4))
    assert lib.semseg_upsample_ce_rmi_table_floats(16, 150) == 16 * 150 * 184 + 4
    assert lib.semseg_upsample_ce_rmi_workspace_floats(2, 33, 33, 21, 3) == -1 and b"zoom 3" in _err()
    assert lib.semseg_upsample_ce_rmi_bwd_workspace_floats(2, 33, 33, 9, 21, 5) == -1 and b"zoom 5" in _err()
    assert lib.semseg_upsample_ce_rmi_table_floats(0, 21) == -1 and b"bad sizes" in _err()
