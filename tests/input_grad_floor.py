"""How well-defined is the input gradient of an eval-mode network at all? The fp32 oracle against ITSELF, on the PSPNet50
65x65, 21-class case of tests/test_input_grad_gpu.py (frozen parameters, cross-entropy against synthetic targets):
  * the input perturbed by 1e-6 relative (x * (1 + 1e-6 n), n ~ N(0, 1));
  * the input perturbed at the scale of bf16x3's operand rounding (2^-17 relative);
  * another summation order: the same network in float64.
A ReLU mask near zero that flips moves a whole path of the gradient, so x.grad is only as well-defined as these
numbers; the network-level tolerance of the GPU tier (INPUT_GRAD_TOL) is set from them."""
import torch
import torch.nn.functional as F

from tests import util

# rel-L2 bound of x.grad (bf16x3) against the fp32 oracle: 3x the floor at bf16x3's operand-rounding scale (measured
# 9.5e-3: at 2^-17 the masks already flip, while 1e-6 and float64 agree to ~1e-6); tests/test_input_grad_cpu.py
# re-measures the floor and checks the bound against it
INPUT_GRAD_TOL = 3e-2


def oracle_input_grad(orc, x, y):
    xg = x.detach().clone().requires_grad_(True)
    F.cross_entropy(orc.forward(xg), y, ignore_index=255).backward()
    return xg.grad


def frozen_eval_oracle(model, arch, dtype=torch.float32, **kw):
    """The oracle of `model` in eval mode with parameters that need no gradient (the attack set-up)."""
    from oracle.torch_oracle import Oracle
    sd = {k: v.detach().clone().to(dtype) if v.is_floating_point() else v.detach().clone()
          for k, v in model.state_dict().items()}
    return Oracle(sd, arch=arch, **kw).eval()


def measure_floor(device="cpu", seed=0):
    """-> (rel-L2 of x.grad under a 1e-6 relative input perturbation, under a 2^-17 one, fp32 against float64)."""
    model = util.build_pspnet(50, 21).to(device).eval()
    orc = frozen_eval_oracle(model, "psp", layers=50, classes=21)
    x, y = util.synth(2, 65, 65, 21, seed=seed, device=device)
    g0 = oracle_input_grad(orc, x, y)
    gen = torch.Generator().manual_seed(seed + 1)
    n = torch.randn(x.shape, generator=gen).to(device)
    out = [util.rel_l2(oracle_input_grad(orc, x * (1 + rel * n), y), g0) for rel in (1e-6, 2.0 ** -17)]
    o64 = frozen_eval_oracle(model, "psp", torch.float64, layers=50, classes=21)
    out.append(util.rel_l2(g0, oracle_input_grad(o64, x.double(), y)))
    return tuple(out)


if __name__ == "__main__":
    print("oracle x.grad floor (rel-L2): 1e-6 perturbation %.3e, 2^-17 perturbation %.3e, fp32 vs float64 %.3e"
          % measure_floor())
