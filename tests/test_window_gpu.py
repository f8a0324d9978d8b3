"""GPU tier for sliding-window evaluation on the native kernels (csrc/window.cu, semseg_b200/inference.py exact=False):
each kernel against the ATen steps it replaces, and the whole engine against the same network behind a wrapper that
forces the ATen path."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import util

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _strict_fp32():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield


def _aten_scores(logits_nhwc, crop, flip):
    """The ATen chain of SlidingWindowPredictor._scores on the model's NCHW eval logits."""
    x = logits_nhwc.permute(0, 3, 1, 2).contiguous()
    prob = F.softmax(F.interpolate(x, (crop, crop), mode="bilinear", align_corners=True), dim=1)
    if flip:
        n = x.shape[0] // 2
        prob = (prob[:n] + prob[n:].flip(3)) / 2
    return prob


# (crop, classes, crops G, extra channels of the logits' pixel pitch, logit scale); logits in the thousands, as an
# untrained PSPNet101 produces, make the softmax sensitive to every rounding of v - max
SCORE_CASES = [(65, 7, 3, 0, 4.0), (473, 150, 1, 0, 4.0), (713, 19, 1, 0, 4.0), (65, 256, 2, 0, 4.0),
               (129, 19, 2, 5, 4.0), (713, 19, 1, 0, 1000.0)]


@pytest.mark.parametrize("case", SCORE_CASES)
@pytest.mark.parametrize("flip", [True, False])
def test_window_scores_match_aten_chain(case, flip):
    from semseg_b200 import ops
    crop, c, g, pad, scale = case
    h = (crop - 1) // 8 + 1
    gen = torch.Generator(device="cuda").manual_seed(crop * 1000 + c + int(flip))
    n = 2 * g if flip else g
    buf = torch.randn((n, h, h, c + pad), device="cuda", generator=gen) * scale
    logits = buf[..., :c]                                   # channel slice: pixel pitch c + pad
    out = torch.full((g + 1, c, crop, crop), -1.0, device="cuda")
    ops.window_scores(logits, flip, out[1:])                # written at a crop offset of a larger score buffer
    torch.cuda.synchronize()
    ref = _aten_scores(logits, crop, flip)
    assert bool((out[0] == -1.0).all())
    got = out[1:]
    assert float((got - ref).abs().max()) <= 1e-6
    assert float((got.sum(1) - 1.0).abs().max()) <= 1e-5


def _loop_canvas(scores, ys, xs, full, top, left, img):
    """The ATen accumulation of SlidingWindowPredictor._scale_canvas."""
    ch, cw = scores.shape[2:]
    canvas = torch.zeros((scores.shape[1],) + tuple(full), dtype=torch.float64, device=scores.device)
    hits = np.zeros(full, dtype=np.float64)
    for k, (y0, x0) in enumerate([(y0, x0) for y0 in ys for x0 in xs]):
        canvas[:, y0:y0 + ch, x0:x0 + cw] += scores[k]
        hits[y0:y0 + ch, x0:x0 + cw] += 1
    canvas /= torch.from_numpy(hits).to(scores.device)
    return canvas[:, top:top + img[0], left:left + img[1]]


# (image h, w, crop, classes): 110 = crop + stride + 1 (three crops overlap on that axis, up to 9 per pixel),
# 50 x 40 is padded to the crop
ACC_CASES = [(110, 200, 65, 7), (110, 110, 65, 19), (50, 40, 65, 7), (300, 40, 65, 5), (800, 713, 713, 19)]


@pytest.mark.parametrize("case", ACC_CASES)
def test_window_accumulate_bit_identical_to_loop(case):
    from semseg_b200 import inference, ops
    img_h, img_w, crop, c = case
    full_h, full_w = max(img_h, crop), max(img_w, crop)
    top, left = (full_h - img_h) // 2, (full_w - img_w) // 2
    ys, xs = inference.crop_origins(full_h, crop), inference.crop_origins(full_w, crop)
    gen = torch.Generator(device="cuda").manual_seed(img_h + img_w + c)
    scores = torch.softmax(torch.randn((len(ys) * len(xs), c, crop, crop), device="cuda", generator=gen), 1)
    got = ops.window_accumulate(scores, ys, xs, (full_h, full_w), top, left, (img_h, img_w))
    ref = _loop_canvas(scores, ys, xs, (full_h, full_w), top, left, (img_h, img_w))
    assert got.shape == ref.shape and torch.equal(got, ref)
    if img_h == crop + int(np.ceil(crop * 2 / 3)) + 1:
        assert len(ys) == 3 and ys[2] - ys[1] == 1          # the clamped last crop: a triple overlap


@pytest.mark.parametrize("src,dst", [((37, 53), (100, 150)), ((200, 300), (100, 150)), ((100, 150), (100, 150)),
                                     ((75, 113), (100, 150)), ((473, 631), (512, 683))])
def test_window_resize_add_matches_interpolate(src, dst):
    from semseg_b200 import ops
    gen = torch.Generator(device="cuda").manual_seed(src[0] * 7 + dst[1])
    c = 19
    canvas = torch.rand((c,) + src, dtype=torch.float64, device="cuda", generator=gen)
    total = torch.rand((c,) + dst, dtype=torch.float64, device="cuda", generator=gen)
    ref = total + F.interpolate(canvas[None], size=dst, mode="bilinear", align_corners=False)[0]
    ops.window_resize_add(canvas, total)
    assert float((total - ref).abs().max() / ref.abs().max()) <= 1e-12


class _Foreign(torch.nn.Module):
    """Same network behind a module the engine does not recognise: forces the ATen finish."""

    def __init__(self, net):
        super().__init__()
        self.net = net

    def forward(self, x):
        return self.net(x)


def _raise(*args, **kwargs):
    raise AssertionError("the native path must not call ATen interpolate / softmax")


@pytest.mark.parametrize("arch", ["psp", "psa"])
def test_engine_native_matches_aten_finish(arch, monkeypatch):
    from semseg_b200 import inference
    c = util.SW_CFG
    classes, crop = 7, 65
    model = (util.build_pspnet(50, classes=classes) if arch == "psp" else util.build_psanet(50, classes=classes))
    model = model.cuda().eval()
    image = util.sw_image(seed=11, h=100, w=150)
    scales, base = [0.4, 0.75, 1.0, 1.25], 150                  # 0.4: a 40 x 60 image, padded to the crop
    aten = inference.SlidingWindowPredictor(_Foreign(model), classes, crop, crop, c["mean"], c["std"], max_batch=8)
    ref_scores, ref_amax = aten(image, base, scales)
    native = inference.SlidingWindowPredictor(model, classes, crop, crop, c["mean"], c["std"], max_batch=8)
    dp = inference.SlidingWindowPredictor(torch.nn.DataParallel(model, device_ids=[0]), classes, crop, crop, c["mean"],
                                          c["std"], max_batch=8)
    with monkeypatch.context() as mp:
        mp.setattr(inference.F, "interpolate", _raise)
        mp.setattr(inference.F, "softmax", _raise)
        scores, amax = native(image, base, scales)
        dp_scores, dp_amax = dp(image, base, scales)
    assert native.forward_calls == aten.forward_calls
    assert scores.shape == ref_scores.shape == (100, 150, classes)
    assert np.abs(scores - ref_scores).max() <= 2e-6
    top2 = np.sort(ref_scores, axis=2)[..., -2:]
    clear = (top2[..., 1] - top2[..., 0]) > 4e-6
    assert clear.mean() > 0.9 and np.array_equal(amax[clear], ref_amax[clear])
    assert np.array_equal(dp_scores, scores) and np.array_equal(dp_amax, amax)
