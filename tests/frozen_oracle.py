"""fp32 oracle of a training network whose named BatchNorm layers are frozen (in eval mode while the network trains):
those layers normalise with their running statistics, which stay untouched together with num_batches_tracked, exactly
like torch's nn.BatchNorm2d / nn.SyncBatchNorm in eval mode. Every other layer behaves as in oracle/torch_oracle.py."""
import torch.nn.functional as F

from oracle.torch_oracle import EPS, MOMENTUM, Oracle


class FrozenBNOracle(Oracle):
    """Oracle with `frozen`: names of BatchNorm layers as in the state_dict (e.g. 'layer1.0.bn1', 'cls.1')."""

    def __init__(self, sd, frozen=(), **kw):
        super().__init__(sd, **kw)
        self.frozen = frozenset(frozen)

    def bn(self, x, name):
        if not (self.training and name in self.frozen):
            return super().bn(x, name)
        sd = self.sd
        return F.batch_norm(x, sd[name + '.running_mean'], sd[name + '.running_var'], sd[name + '.weight'],
                            sd[name + '.bias'], False, MOMENTUM, EPS)


def frozen_oracle_from(model, arch, frozen=(), **kw):
    """FrozenBNOracle sharing (clones of) the model's parameters and buffers (tests/util.py::oracle_from)."""
    params = {k for k, _ in model.named_parameters()}
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    for k, v in sd.items():
        if k in params:
            v.requires_grad_(True)
    return FrozenBNOracle(sd, frozen=frozen, arch=arch, **kw), sd
