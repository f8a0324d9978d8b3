"""CPU tier for the relation term of losses.DistillationLoss (csrc/relation.cu): option validation and extra_repr,
the C entry points' argument checks (SEMSEG_E_INVALID before any CUDA call), and properties of the float64 oracle of
tests/relation_oracle.py, its closed-form gradient against autograd included."""
import ctypes
import math

import pytest
import torch

from semseg_b200 import _lib
from semseg_b200.losses import DistillationLoss
from tests import util
from tests.relation_oracle import relation_grad, relation_loss, relation_loss_nodes

P = ctypes.c_void_p(16)      # never dereferenced: validation fails before any launch
E_INVALID = -1


def _err():
    return _lib.load().semseg_last_error()


@pytest.fixture(scope="module")
def nets():
    return util.build_pspnet(50, 21), util.build_pspnet(50, 21, seed=1).eval()


# ------------------------------------------------------------------------------------------------ options
def test_relation_options_validation_and_repr(nets):
    teacher = nets[1]
    d = DistillationLoss(teacher)
    assert (d.relation_weight, d.relation_temperature, d.relation_pool) == (0.0, 1.0, 2)
    assert "relation" not in repr(d)
    c = DistillationLoss(teacher, relation_weight=2, relation_temperature=0.5, relation_pool=3)
    assert isinstance(c.relation_weight, float) and c.relation_weight == 2.0
    assert "relation_weight=2, relation_temperature=0.5, relation_pool=3" in repr(c)
    assert "relation" not in repr(DistillationLoss(teacher, relation_temperature=0.5, relation_pool=3))
    for kw in ({"relation_weight": True}, {"relation_weight": "1"}, {"relation_weight": None},
               {"relation_temperature": False}, {"relation_temperature": "1"}, {"relation_pool": True},
               {"relation_pool": 2.0}, {"relation_pool": "2"}, {"relation_pool": None}):
        with pytest.raises(TypeError):
            DistillationLoss(teacher, **kw)
    for kw in ({"relation_weight": -0.1}, {"relation_weight": float("nan")}, {"relation_weight": float("inf")},
               {"relation_temperature": 0.0}, {"relation_temperature": -1.0},
               {"relation_temperature": float("inf")}, {"relation_temperature": float("nan")},
               {"relation_pool": 0}, {"relation_pool": -1}, {"relation_pool": 17}):
        with pytest.raises(ValueError):
            DistillationLoss(teacher, **kw)


def test_last_relation_is_none_before_a_forward(nets):
    assert DistillationLoss(nets[1]).last_relation() is None
    assert DistillationLoss(nets[1], relation_weight=1.0).last_relation() is None


# ------------------------------------------------------------------------------------------------ C-ABI validation
def _nodes(**kw):
    a = dict(feat=P, feat_lo=None, pitch=512, B=2, h=9, w=13, C=512, pool=2, nodes=P, nodes_lo=None, arg=None,
             inv=None)
    a.update(kw)
    return _lib.load().semseg_relation_nodes(a["feat"], a["feat_lo"], a["pitch"], a["B"], a["h"], a["w"], a["C"],
                                             a["pool"], a["nodes"], a["nodes_lo"], a["arg"], a["inv"], None)


def _kl(fn, **kw):
    a = dict(xs=P, xs_lo=None, xt=P, xt_lo=None, B=2, M=35, C=512, tau=1.0, p0=P, p1=P, p2=P)
    a.update(kw)
    return getattr(_lib.load(), fn)(a["xs"], a["xs_lo"], a["xt"], a["xt_lo"], a["B"], a["M"], a["C"], a["tau"],
                                    a["p0"], a["p1"], a["p2"], None)


def _nodes_bwd(**kw):
    a = dict(feat=P, feat_lo=None, pitch=512, B=2, h=9, w=13, C=512, pool=2, arg=P, inv=P, dn=P, df=P, df_lo=None,
             dfp=512)
    a.update(kw)
    return _lib.load().semseg_relation_nodes_bwd(a["feat"], a["feat_lo"], a["pitch"], a["B"], a["h"], a["w"], a["C"],
                                                 a["pool"], a["arg"], a["inv"], a["dn"], a["df"], a["df_lo"], a["dfp"],
                                                 None)


@pytest.mark.parametrize("kw", [dict(feat=None), dict(nodes=None), dict(B=0), dict(h=0), dict(w=-1), dict(C=256),
                                dict(pool=0), dict(pool=17), dict(pitch=516), dict(pitch=504),
                                dict(feat=ctypes.c_void_p(24)), dict(nodes=ctypes.c_void_p(24)),
                                dict(arg=P), dict(inv=P), dict(arg=ctypes.c_void_p(24), inv=P)])
def test_nodes_entry_point_validates(kw):
    assert _nodes(**kw) == E_INVALID
    assert b"relation_nodes" in _err()


@pytest.mark.parametrize("fn", ["semseg_relation_kl_fwd", "semseg_relation_kl_bwd"])
@pytest.mark.parametrize("kw", [dict(xs=None), dict(xt=None), dict(B=0), dict(M=0), dict(C=256), dict(tau=0.0),
                                dict(tau=-1.0), dict(tau=float("inf")), dict(tau=float("nan")), dict(xs_lo=P),
                                dict(xs=ctypes.c_void_p(24)), dict(xt=ctypes.c_void_p(8)),
                                dict(xs_lo=ctypes.c_void_p(40), xt_lo=P), dict(p0=None), dict(p1=None), dict(p2=None),
                                dict(p0=ctypes.c_void_p(20)), dict(B=4096, M=4096)])
def test_kl_entry_points_validate(fn, kw):
    assert _kl(fn, **kw) == E_INVALID
    assert fn[len("semseg_"):].encode() in _err()


@pytest.mark.parametrize("kw", [dict(feat=None), dict(arg=None), dict(inv=None), dict(dn=None), dict(df=None),
                                dict(C=128), dict(pool=0), dict(pool=20), dict(pitch=12), dict(dfp=516),
                                dict(dfp=256), dict(arg=ctypes.c_void_p(8)), dict(df=ctypes.c_void_p(24))])
def test_nodes_bwd_entry_point_validates(kw):
    assert _nodes_bwd(**kw) == E_INVALID
    assert b"relation_nodes_bwd" in _err()


def test_workspace_size():
    lib = _lib.load()
    assert lib.semseg_relation_workspace_floats(16, 900) == 2 * 16 * 16 * 15
    assert lib.semseg_relation_workspace_floats(0, 900) == -1
    assert lib.semseg_relation_workspace_floats(2, 0) == -1


# ------------------------------------------------------------------------------------------------ oracle properties
def _feat(seed, b=3, h=7, w=9, c=16):
    g = torch.Generator().manual_seed(seed)
    f = torch.relu(torch.randn((b, h, w, c), generator=g, dtype=torch.float64))
    f[0, :2, :2] = 0.0                                  # an all-zero node at pool 2
    return f


@pytest.mark.parametrize("pool", [1, 2, 3])
@pytest.mark.parametrize("tau", [0.1, 1.0, 4.0])
def test_oracle_closed_form_gradient_equals_autograd(pool, tau):
    fs, ft = _feat(1), _feat(2)
    fr = fs.clone().requires_grad_(True)
    (g,) = torch.autograd.grad(relation_loss(fr, ft, tau, pool), fr)
    g_cf = relation_grad(fs, ft, tau, pool)
    assert float((g - g_cf).abs().max()) <= 1e-12 * max(1.0, float(g.abs().max()))
    if pool == 2:
        assert float(g_cf[0, :2, :2].abs().max()) == 0.0       # the zero node gets no gradient


def test_oracle_rounded_gradient_equals_autograd():
    fs, ft = _feat(3), _feat(4)
    fr = fs.clone().requires_grad_(True)
    (g,) = torch.autograd.grad(relation_loss(fr, ft, 1.0, 2, round_nodes=True), fr)
    g_cf = relation_grad(fs, ft, 1.0, 2, round_nodes=True)
    assert float((g - g_cf).abs().max()) <= 1e-12 * max(1.0, float(g.abs().max()))


def test_oracle_batch_permutation_invariance():
    fs, ft = _feat(5, b=4), _feat(6, b=4)
    perm = torch.tensor([2, 0, 3, 1])
    r = relation_loss(fs, ft, 0.5, 2)
    rp = relation_loss(fs[perm], ft[perm], 0.5, 2)
    assert math.isclose(float(r), float(rp), rel_tol=1e-12)
    g, gp = relation_grad(fs, ft, 0.5, 2), relation_grad(fs[perm], ft[perm], 0.5, 2)
    assert float((g[perm] - gp).abs().max()) <= 1e-14


def test_oracle_identical_nodes_give_zero():
    fs = _feat(7)
    assert abs(float(relation_loss(fs, fs.clone(), 1.0, 2))) <= 1e-15
    assert float(relation_grad(fs, fs.clone(), 1.0, 2).abs().max()) <= 1e-15
    assert float(relation_loss(fs, 2.5 * fs, 1.0, 2)) <= 1e-15        # normalisation removes the scale


def test_oracle_single_node_gives_zero():
    g = torch.Generator().manual_seed(8)
    xs = torch.randn((3, 1, 16), generator=g, dtype=torch.float64)
    xt = torch.randn((3, 1, 16), generator=g, dtype=torch.float64)
    assert float(relation_loss_nodes(xs, xt, 1.0)) == 0.0
    fs, ft = _feat(9, h=2, w=2), _feat(10, h=2, w=2)
    assert float(relation_loss(fs, ft, 1.0, 2)) == 0.0
