"""GPU tier for Monte Carlo dropout (semseg_b200/inference.py with mc_draws > 0, csrc/window.cu's
semseg_window_scores_mc): the kernel against the float64 oracle (tests/mc_oracle.py) and against the plain scores
kernel at T = 1, the native per-draw logits against the eval forward with cls[3] in training mode, and the native
predictor against its ATen path over the same network under one seed."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from semseg_b200 import ops, precision
from semseg_b200.inference import SlidingWindowPredictor
from tests import mc_oracle as O
from tests import util

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _strict_fp32():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield


# ------------------------------------------------------------------------------------------------ kernel
# (crop, classes, crops G, extra channels of the logits' pixel pitch); crops 65, 97 and 129 leave a partial 64-column CTA
CASES = [(65, 19, 3, 0), (97, 150, 2, 3), (129, 256, 1, 0), (713, 19, 1, 0), (129, 19, 2, 5)]


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("draws", [1, 3, 20])
@pytest.mark.parametrize("flip", [True, False])
@pytest.mark.parametrize("gain", [4.0, 100.0], ids=["x4", "x100"])
def test_window_scores_mc_matches_oracle(case, draws, flip, gain):
    crop, c, g, pad = case
    h = (crop - 1) // 8 + 1
    n = 2 * g if flip else g
    gen = torch.Generator(device="cuda").manual_seed(crop * 31 + c + 7 * draws + int(flip))
    logits = (torch.randn((draws, n, h, h, c + pad), device="cuda", generator=gen) * gain)[..., :c]
    out = ops.window_scores_mc(logits, flip, torch.full((g, c + 1, crop, crop), float("nan"), device="cuda"))
    again = ops.window_scores_mc(logits, flip, torch.empty((g, c + 1, crop, crop), device="cuda"))
    torch.cuda.synchronize()
    assert torch.equal(out, again)
    if draws == 1:
        plain = ops.window_scores(logits[0], flip, torch.empty((g, c, crop, crop), device="cuda"))
        assert torch.equal(out[:, :c], plain)
    ref = O.mc_scores(logits, flip)
    err_p = float((out[:, :c].double() - ref[:, :c]).abs().max())
    err_h = float((out[:, c].double() - ref[:, c]).abs().max())
    # the same softmax and entropy in fp64 from ATen's fp32 upsample of the logits (lerp_aten's rounding)
    ref32 = O.mc_scores(logits, flip, upsample=lambda lt: F.interpolate(
        lt.permute(0, 3, 1, 2).contiguous(), (crop, crop), mode="bilinear", align_corners=True))
    err_p32 = float((out[:, :c].double() - ref32[:, :c]).abs().max())
    # An interpolated fp32 logit carries up to 3 roundings of |v| 2^-24 each, and a score moves by at most
    # q (1 - q) <= 1/4 times a logit error: the exact scores are within |v|max 2^-24 of fp32-interpolated ones. At x4
    # that is < 2e-6; at x100 (|v| near 500) it is ~3e-5 and dominates. window_scores has the same error, bit for bit.
    vmax = float(logits.abs().max())
    assert err_p32 <= 2e-6 and err_p <= 2e-6 + vmax * 2.0 ** -24 and err_h <= 1e-5 * max(1.0, float(np.log(c))), \
        (err_p32, err_p, err_h, vmax)


# ------------------------------------------------------------------------------------------------ per-draw logits
def _model(arch, classes=7, p=0.3):
    m = util.build_pspnet(50, classes=classes) if arch == "psp" else util.build_psanet(50, classes=classes)
    m.cls[3].p = p
    m.aux[3].p = p
    return m.cuda().eval()


@pytest.mark.parametrize("arch", ["psp", "psa"])
@pytest.mark.parametrize("mode", ["bf16", "bf16x3"])
def test_native_draws_equal_eval_forward_with_training_dropout(arch, mode):
    net = _model(arch)
    x = torch.randn((4, 3, 65, 65), device="cuda", generator=torch.Generator(device="cuda").manual_seed(3)) * 50
    draws = 4
    with precision.mode(mode), torch.no_grad():
        torch.manual_seed(11)
        got = net._mc_eval_logits_nhwc(x, draws)
        torch.manual_seed(11)
        net.cls[3].train()
        try:
            refs = [net._eval_logits_nhwc(x) for _ in range(draws)]
        finally:
            net.cls[3].eval()
        plain = net._eval_logits_nhwc(x)
    assert tuple(got.shape) == (draws,) + tuple(refs[0].shape)
    for t in range(draws):
        assert torch.equal(got[t], refs[t]), t
    assert not torch.equal(got[0], got[1]) and not torch.equal(got[0], plain)


# ------------------------------------------------------------------------------------------------ predictor
class _Foreign(torch.nn.Module):
    """Same network behind a module the engine does not recognise: forces the ATen path."""

    def __init__(self, net):
        super().__init__()
        self.net = net

    def forward(self, x):
        return self.net(x)


def _make(model, **kw):
    c = util.SW_CFG
    return SlidingWindowPredictor(model, 7, 65, 65, c["mean"], c["std"], max_batch=8, **kw)


def _run(pred, image, seed, base, scales, **kw):
    torch.manual_seed(seed)
    return pred(image, base, scales, **kw)


@pytest.mark.parametrize("arch", ["psp", "psa"])
@pytest.mark.parametrize("scales", [[1.0], [0.4, 0.75, 1.0, 1.25]])
def test_native_predictor_matches_aten_path(arch, scales):
    model = _model(arch)
    image = util.sw_image(seed=21, h=100, w=150)
    base, draws = 150, 5
    native = _make(model, mc_draws=draws)
    s_n, a_n, u_n = _run(native, image, 4, base, scales)
    aten = _make(_Foreign(model), mc_draws=draws)
    s_a, a_a, u_a = _run(aten, image, 4, base, scales)
    assert aten.forward_calls == draws * native.forward_calls
    assert not model.cls[3].training and not model.aux[3].training
    assert float(np.abs(s_n - s_a).max()) <= 2e-5
    top2 = np.sort(s_n, axis=2)[..., -2:]
    sure = (top2[..., 1] - top2[..., 0]) > 1e-5
    assert np.array_equal(a_n[sure], a_a[sure])
    assert u_n.is_cuda and u_n.dtype == torch.float32 and tuple(u_n.shape) == (2, 100, 150)
    for k in range(2):
        span = float(u_n[k].abs().max())
        assert float((u_n[k] - u_a[k]).abs().max()) <= 2e-5 * max(1.0, span), k
    assert float(u_n[1].min()) >= -1e-5
    assert float(u_n[1].max()) > 0.0             # dropout at p = 0.3 moves the predictions
    # the finish is the contract's, on the predictor's own total
    torch.manual_seed(4)
    total, _ = _make(model, mc_draws=draws)._stats_total(image, base, scales, mc=True)
    ref = O.uncertainty(total, 7)
    assert float((u_n.double() - ref).abs().max()) <= 1e-6


def test_native_predictor_is_deterministic_and_counts_one_call_per_batch():
    model = _model("psp")
    image = util.sw_image(seed=22, h=100, w=150)
    scales = [0.75, 1.0]
    runs = []
    for _ in range(2):
        p = _make(model, mc_draws=3)
        runs.append(_run(p, image, 9, 150, scales))
        ref = _make(model)
        ref(image, 150, scales)
        assert p.forward_calls == ref.forward_calls
    (s1, a1, u1), (s2, a2, u2) = runs
    assert np.array_equal(s1, s2) and np.array_equal(a1, a2) and torch.equal(u1, u2)
    s3, _, u3 = _run(_make(model, mc_draws=3), image, 10, 150, scales)
    assert not np.array_equal(s1, s3) and not torch.equal(u1, u3)
    assert np.abs(s1.sum(2) - 1.0).max() <= 1e-5


def test_mc_draws_zero_is_the_deterministic_predictor():
    model = _model("psp")
    image = util.sw_image(seed=23, h=100, w=150)
    s0, a0 = _make(model)(image, 150, [0.75, 1.0])
    s1, a1 = _make(model, mc_draws=0)(image, 150, [0.75, 1.0])
    assert np.array_equal(s0, s1) and np.array_equal(a0, a1)
