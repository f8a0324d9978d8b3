"""CPU tier: the criterion's part of the key of a captured training step (graphs.train_step). Every option a criterion
bakes into the step's graphs is in the key, so a changed option captures anew rather than replaying a stale graph; an
option that launches nothing (the relation term's options at relation_weight 0, streams=1) leaves the key alone. The teacher of a
distillation or pseudo-label criterion enters by identity and, unless it is a ModelEMA shadow, by its tensors'
versions; the class weights by their tensor's address."""
import pytest
import torch
from torch import nn

from semseg_b200 import graphs
from semseg_b200.augment import StrongAugment
from semseg_b200.losses import (DiceLoss, DistillationLoss, EntropyLoss, FocalLoss, GatedCRFLoss, LovaszSoftmaxLoss,
                                MixPseudoLabelLoss, OhemCrossEntropyLoss, PseudoLabelLoss, RMILoss)
from semseg_b200.optim import ModelEMA
from tests import util

TEACHER_CRITERIA = (DistillationLoss, PseudoLabelLoss, MixPseudoLabelLoss)
W1, W2 = torch.ones(21), torch.ones(21)          # two class-weight tensors of equal values, different storage
STRONG = StrongAugment()


@pytest.fixture(scope="module")
def nets():
    return util.build_pspnet(50, 21), util.build_pspnet(50, 21, seed=1).eval()


@pytest.fixture
def crit_key(nets, monkeypatch):
    """crit_key(criterion): the criterion part (the last entry) of the key graphs.train_step builds for the student
    with that criterion, taken where the step would be created."""
    student = nets[0]
    keys = []

    class _Stop(Exception):
        pass

    def fake_step(key):
        keys.append(key)
        raise _Stop

    monkeypatch.setattr(graphs, "_Step", fake_step)
    monkeypatch.setattr(graphs, "enabled", lambda: True)
    y = torch.zeros((1, 17, 17), dtype=torch.int64)

    class _X:
        """A stand-in input that passes train_step's device test."""
        is_cuda, shape, dtype, requires_grad = True, torch.Size((1, 3, 17, 17)), torch.float32, False
        device = torch.device("cuda", 0)

    def key(criterion):
        student.criterion = criterion
        student.__dict__.pop("_sb_graph_steps", None)
        with pytest.raises(_Stop):
            graphs.train_step(student, None, _X(), y)
        return keys[-1][-1]

    old = student.criterion
    yield key
    student.criterion = old


def _strong(**kw):
    return dict(strong=StrongAugment(**kw))


# (criterion class, base arguments, variants of the base, partition): variant i is the criterion built with the base
# updated by variants[i]; two variants have the same key exactly when their partition labels are equal
CASES = {
    "ce": (nn.CrossEntropyLoss, dict(ignore_index=255),
           [dict(), dict(ignore_index=0), dict(label_smoothing=0.1), dict(label_smoothing=0.2), dict(reduction='sum'),
            dict(weight=W1), dict(weight=W1), dict(weight=W2)],
           [0, 1, 2, 3, 4, 5, 5, 6]),
    "ohem": (OhemCrossEntropyLoss, dict(),
             [dict(), dict(ignore_index=0), dict(thresh=0.5), dict(min_kept=1000), dict(weight=W1), dict(weight=W1),
              dict(weight=W2)],
             [0, 1, 2, 3, 4, 4, 5]),
    "dice": (DiceLoss, dict(),
             [dict(), dict(ignore_index=0), dict(smooth=1.0), dict(eps=1e-5), dict(ce_weight=1.0)],
             [0, 1, 2, 3, 4]),
    "focal": (FocalLoss, dict(),
              [dict(), dict(ignore_index=0), dict(gamma=0.0), dict(gamma=1.0), dict(weight=W1), dict(weight=W1),
               dict(weight=W2)],
              [0, 1, 2, 3, 4, 4, 5]),
    "entropy": (EntropyLoss, dict(),
                [dict(), dict(ignore_index=0), dict(ent_weight=0.5), dict(ce_weight=0.0)],
                [0, 1, 2, 3]),
    "gatedcrf": (GatedCRFLoss, dict(),
                 [dict(), dict(ignore_index=0), dict(crf_weight=0.2), dict(ce_weight=0.5), dict(radius=3),
                  dict(sigma_xy=3.0), dict(sigma_rgb=0.2), dict(at='logits'), dict(mean=(0.0, 0.0, 0.0)),
                  dict(std=(1.0, 1.0, 1.0))],
                 list(range(10))),
    "lovasz": (LovaszSoftmaxLoss, dict(),
               [dict(), dict(ignore_index=0), dict(classes='all'), dict(per_image=True), dict(ce_weight=1.0)],
               [0, 1, 2, 3, 4]),
    "rmi": (RMILoss, dict(),
            [dict(), dict(ignore_index=0), dict(bce_weight=0.2), dict(pos_alpha=1e-3), dict(ce_weight=1.0)],
            [0, 1, 2, 3, 4]),
    "kd": (DistillationLoss, dict(),
           [dict(), dict(ignore_index=0), dict(temperature=2.0), dict(kd_weight=0.5), dict(ce_weight=0.0),
            dict(at='logits')],
           [0, 1, 2, 3, 4, 5]),
    # the relation term's options count only when it runs: at weight 0 the key is the one without them
    "relation": (DistillationLoss, dict(),
                 [dict(), dict(relation_weight=0.0, relation_temperature=4.0, relation_pool=3),
                  dict(relation_weight=1.0), dict(relation_weight=0.5),
                  dict(relation_weight=1.0, relation_temperature=4.0), dict(relation_weight=1.0, relation_pool=1)],
                 [0, 0, 1, 2, 3, 4]),
    "pl": (PseudoLabelLoss, dict(),
           [dict(), dict(ignore_index=0), dict(threshold=0.5), dict(pl_weight=0.5), dict(ce_weight=0.5)],
           [0, 1, 2, 3, 4]),
    "mix": (MixPseudoLabelLoss, dict(),
            [dict(), dict(mix='classmix'), dict(p=0.3), dict(area=(0.1, 0.4)), dict(ratio=(0.5, 2.0)),
             dict(threshold=0.5)],
            [0, 1, 2, 3, 4, 5]),
}
# the feature perturbation: each option is launched, fp_dropout alone included
FP_VARIANTS = ([dict(), dict(fp_weight=0.5), dict(fp_weight=0.25), dict(fp_weight=0.5, fp_dropout=0.3),
                dict(fp_weight=0.5, fp_dropout=0.0), dict(fp_dropout=0.3)], [0, 1, 2, 3, 4, 5])
# two streams are a 2N-image student; streams=1 is the default's key
DUAL_VARIANTS = ([dict(), dict(streams=1), dict(streams=2), dict(streams=2, fp_weight=0.5), dict(fp_weight=0.5)],
                 [0, 0, 1, 2, 3])
# every option of the strong view; without a view (strong=None, the default) the key is the criterion's own
STRONG_VARIANTS = ([dict(), dict(strong=None), _strong(), _strong(brightness=0.4), _strong(contrast=0.4),
                    _strong(saturation=0.4), _strong(hue=0.2), _strong(p_jitter=0.7), _strong(p_gray=0.1),
                    _strong(p_blur=0.4), _strong(sigma=(0.2, 2.0)), _strong(sigma=(0.1, 3.0)),
                    _strong(mean=(1.0, 2.0, 3.0)), _strong(std=(50.0, 60.0, 70.0))],
                   [0, 0] + list(range(1, 13)))
for cls in (PseudoLabelLoss, MixPseudoLabelLoss):
    CASES["fp_" + cls.__name__] = (cls, dict()) + FP_VARIANTS
    CASES["dual_" + cls.__name__] = (cls, dict(strong=STRONG)) + DUAL_VARIANTS
for cls in TEACHER_CRITERIA:
    CASES["strong_" + cls.__name__] = (cls, dict()) + STRONG_VARIANTS


@pytest.mark.parametrize("case", list(CASES))
def test_options_enter_the_graph_key(case, nets, crit_key):
    cls, base, variants, partition = CASES[case]
    assert len(variants) == len(partition)
    head = (nets[1],) if cls in TEACHER_CRITERIA else ()
    keys = [crit_key(cls(*head, **dict(base, **kw))) for kw in variants]
    for i in range(len(keys)):
        for j in range(i):
            assert (keys[i] == keys[j]) == (partition[i] == partition[j]), (variants[j], variants[i])


@pytest.mark.parametrize("cls", TEACHER_CRITERIA)
def test_teacher_enters_the_graph_key(cls, nets, crit_key):
    """Another teacher object is a new key, and so is an in-place edit of a frozen teacher's weight; a ModelEMA shadow
    is keyed by its tensors' addresses only, so the same edit (ema.update) keeps its key."""
    student, teacher = nets
    k = crit_key(cls(teacher))
    assert crit_key(cls(teacher)) == k              # a new criterion with the same options and teacher
    assert "strong" not in k
    other = util.build_pspnet(50, 21, seed=1).eval()
    k_other = crit_key(cls(other))
    assert k_other != k
    with torch.no_grad():
        other.cls[4].weight.mul_(1.5)
    assert crit_key(cls(other)) != k_other
    shadow = ModelEMA(student).module
    k_ema = crit_key(cls(shadow))
    with torch.no_grad():
        shadow.cls[4].weight.mul_(1.5)
    assert crit_key(cls(shadow)) == k_ema


@pytest.mark.parametrize("cls", [nn.CrossEntropyLoss, OhemCrossEntropyLoss, FocalLoss])
def test_class_weight_edit_in_place_keeps_the_graph_key(cls, crit_key):
    w = torch.ones(21)
    crit = cls(weight=w)
    k = crit_key(crit)
    with torch.no_grad():
        w.mul_(2.0)
    assert crit_key(crit) == k
