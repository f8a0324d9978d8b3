"""GPU tier: the reference's validate() call pattern (tool/train.py:353-359) — `model.eval()` then `model(input)` with
autograd ENABLED and every parameter requiring grad, followed by `criterion(output, target)`; nothing is back-propagated.
The eval-mode BatchNorm path folds conv + BN (+ residual, ReLU) into one kernel that has no backward, so it must neither
raise nor change the numbers relative to the torch.no_grad() call that tool/test.py makes."""
import pytest
import torch
import torch.nn.functional as F

from tests import psamask_cases, util

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("arch", ["psp", "psa"])
def test_eval_forward_with_autograd_enabled_equals_no_grad(arch):
    build = util.build_pspnet if arch == "psp" else util.build_psanet
    model = build(50, 21).cuda().eval()
    assert all(p.requires_grad for p in model.parameters())
    x, y = util.synth(2, 65, 65, 21, device="cuda")
    with torch.no_grad():
        ref = model(x)
    assert torch.is_grad_enabled()
    out = model(x)                                   # what validate() does
    assert tuple(out.shape) == tuple(ref.shape) == (2, 21, 65, 65)
    assert bool(torch.isfinite(out).all())
    assert torch.allclose(out.detach(), ref, rtol=0.0, atol=1e-6)
    loss = F.cross_entropy(out, y, ignore_index=255)     # criterion(output, target), tool/train.py:360
    assert bool(torch.isfinite(loss))


def _load_stock_psamask():
    """The reference's own CUDA extension (lib/psa/src/gpu/*), compiled in place by oracle/build.py into oracle/_ref/."""
    import importlib.util
    import os
    ref_dir = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref")
    for f in sorted(os.listdir(ref_dir)) if os.path.isdir(ref_dir) else []:
        if f.startswith("psamask_ref_gpu") and f.endswith(".so"):
            spec = importlib.util.spec_from_file_location("psamask_ref_gpu", os.path.join(ref_dir, f))
            mod = importlib.util.module_from_spec(spec)
            spec.loader.exec_module(mod)
            return mod
    return None


@pytest.mark.parametrize("geom", psamask_cases.GPU_GEOMS)
@pytest.mark.parametrize("psa_type", [0, 1])
def test_psamask_bit_identical_to_the_references_cuda_kernel(geom, psa_type, golden_dir):
    """psa_mask forward / backward against the reference's stock GPU kernel (lib/psa/src/gpu/psamask_cuda.cu:8-128) called
    the way lib/psa/functions/psamask.py:17-35 calls it (zero-filled output, then the kernel): bit-identical. The digests
    of the stock kernel's outputs on these seeded inputs are stored in tests/golden/psamask_ref_digests.json; where
    oracle/_ref holds the compiled extension it is compared live as well."""
    import hashlib
    import json
    import os
    from semseg_b200 import ops
    n, h, w, mh, mw = geom
    key, x_np, go_np = psamask_cases.gpu_case(geom, psa_type)
    dig = json.load(open(os.path.join(golden_dir, "psamask_ref_digests.json")))["gpu"][key]
    x = torch.from_numpy(x_np).cuda()
    go = torch.from_numpy(go_np).cuda()
    got_out = ops.psamask_fwd(x, psa_type, mh, mw)
    got_gin = ops.psamask_bwd(go, psa_type, mh, mw)
    assert hashlib.sha256(got_out.cpu().contiguous().numpy().tobytes()).hexdigest() == dig["out"]
    assert hashlib.sha256(got_gin.cpu().contiguous().numpy().tobytes()).hexdigest() == dig["din"]
    stock = _load_stock_psamask()
    if stock is None:
        return
    out = torch.zeros((n, h * w, h, w), device="cuda")
    stock.psamask_forward(psa_type, x, out, n, h, w, mh, mw, (mh - 1) // 2, (mw - 1) // 2)
    gin = torch.zeros((n, mh * mw, h, w), device="cuda")
    stock.psamask_backward(psa_type, go, gin, n, h, w, mh, mw, (mh - 1) // 2, (mw - 1) // 2)
    torch.cuda.synchronize()
    assert torch.equal(got_out, out)
    assert torch.equal(got_gin, gin)
