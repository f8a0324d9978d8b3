"""GPU tier for anomaly segmentation (semseg_b200/anomaly.py, csrc/anomaly.cu, the stats variant of csrc/window.cu):
the stats kernel against the plain scores kernel and the ATen chain, the predictor's scores and argmax against
anomaly=None and its anomaly maps against the ATen finish, the class moments, the SML post-processing and the metrics
against the float64 contract of tests/anomaly_oracle.py."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from semseg_b200 import ops
from semseg_b200.anomaly import AnomalyMeter, AnomalyScorer
from tests import anomaly_oracle as O
from tests import util

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _strict_fp32():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield


# ------------------------------------------------------------------------------------------------ stats kernel
# (crop, classes, crops G, extra channels of the logits' pixel pitch); crops 65, 97 and 129 leave a partial 64-column CTA
STATS_CASES = [(65, 19, 3, 0), (97, 150, 2, 3), (129, 256, 1, 0), (713, 19, 1, 0), (129, 19, 2, 5)]


@pytest.mark.parametrize("case", STATS_CASES)
@pytest.mark.parametrize("flip", [True, False])
def test_window_scores_stats(case, flip):
    crop, c, g, pad = case
    h = (crop - 1) // 8 + 1
    gen = torch.Generator(device="cuda").manual_seed(crop * 31 + c + int(flip))
    n = 2 * g if flip else g
    logits = (torch.randn((n, h, h, c + pad), device="cuda", generator=gen) * 4.0)[..., :c]
    plain = ops.window_scores(logits, flip, torch.empty((g, c, crop, crop), device="cuda"))
    stats = ops.window_scores(logits, flip, torch.full((g, c + 2, crop, crop), float("nan"), device="cuda"), stats=True)
    torch.cuda.synchronize()
    assert torch.equal(stats[:, :c], plain)
    up = F.interpolate(logits.permute(0, 3, 1, 2).contiguous(), (crop, crop), mode="bilinear", align_corners=True)
    ml, lse = up.amax(1), torch.logsumexp(up, 1)
    if flip:
        ml = (ml[:g] + ml[g:].flip(2)) * 0.5
        lse = (lse[:g] + lse[g:].flip(2)) * 0.5
    assert float((stats[:, c] - ml).abs().max()) <= 2e-6 * float(ml.abs().max())
    assert float((stats[:, c + 1] - lse).abs().max()) <= 4e-6 * float(lse.abs().max())


# ------------------------------------------------------------------------------------------------ predictor
class _Foreign(torch.nn.Module):
    """Same network behind a module the engine does not recognise: forces the ATen finish."""

    def __init__(self, net):
        super().__init__()
        self.net = net

    def forward(self, x):
        return self.net(x)


def _model(arch, classes):
    m = util.build_pspnet(50, classes=classes) if arch == "psp" else util.build_psanet(50, classes=classes)
    return m.cuda().eval()


@pytest.mark.parametrize("arch", ["psp", "psa"])
@pytest.mark.parametrize("scales", [[1.0], [0.4, 0.75, 1.0, 1.25]])
def test_predictor_scores_unchanged_and_maps_match(arch, scales):
    from semseg_b200 import inference
    c = util.SW_CFG
    classes, crop, base = 7, 65, 150
    model = _model(arch, classes)
    images = [util.sw_image(seed=s, h=100, w=150) for s in (11, 12)]
    make = lambda m, a=None: inference.SlidingWindowPredictor(m, classes, crop, crop, c["mean"], c["std"],  # noqa: E731
                                                                 max_batch=8, anomaly=a)
    plain = make(model)
    ref_scores, ref_pred = plain(images[0], base, scales)
    fitted = AnomalyScorer("sml").fit(make(model), images, base, scales)
    aten_fitted = AnomalyScorer("sml").fit(make(_Foreign(model)), images, base, scales)
    assert np.allclose(fitted.statistics[0].numpy(), aten_fitted.statistics[0].numpy(), rtol=1e-5, atol=1e-5)
    for kind in ("msp", "maxlogit", "energy", "sml"):
        scorer = AnomalyScorer(kind, statistics=fitted.statistics)
        scores, pred, amap = make(model, scorer)(images[0], base, scales)
        assert np.array_equal(scores, ref_scores) and np.array_equal(pred, ref_pred), kind
        assert amap.is_cuda and amap.dtype == torch.float32 and amap.shape == (100, 150)
        none, pred2, amap2 = make(model, scorer)(images[0], base, scales, return_scores=False)
        assert none is None and np.array_equal(pred2, pred) and torch.equal(amap2, amap)
        a_scores, a_pred, a_map = make(_Foreign(model), scorer)(images[0], base, scales)
        p_scores, p_pred = make(_Foreign(model))(images[0], base, scales)
        assert np.array_equal(a_scores, p_scores) and np.array_equal(a_pred, p_pred), kind
        diff = (amap - a_map).abs().cpu().numpy()
        span = float(amap.abs().max())
        if kind != "sml" or np.array_equal(a_pred, pred):
            assert diff.max() <= 2e-5 * max(span, 1.0), (kind, diff.max())
        else:            # a flipped near-tie moves SML's boundaries: the rest of the map still agrees
            assert (diff <= 2e-5 * max(span, 1.0)).mean() > 0.9, kind
    # the SML map is the contract's, on the predictor's own ML and argmax
    total, pred = make(model)._stats_total(images[0], base, scales)
    mean, std = (t.numpy() for t in fitted.statistics)
    ref = O.sml_map(total[classes].cpu().numpy(), pred.cpu().numpy(), mean, std).astype(np.float32)
    got = AnomalyScorer("sml", statistics=fitted.statistics).score_map(total, pred).cpu().numpy()
    assert np.all(np.abs(got - ref) <= np.spacing(np.abs(ref)) + 1e-13)
    # the fit's statistics are the contract's on the fit pixels
    mls, preds = [], []
    for im in images:
        t, p = make(model)._stats_total(im, base, scales)
        mls.append(t[classes].cpu().numpy())
        preds.append(p.cpu().numpy())
    m_ref, s_ref = O.class_statistics(np.concatenate(preds, None), np.concatenate(mls, None), classes)
    assert np.allclose(fitted.statistics[0].numpy(), m_ref, rtol=1e-12, atol=1e-12)
    assert np.allclose(fitted.statistics[1].numpy(), s_ref, rtol=1e-7, atol=1e-9)


def test_sml_without_statistics_raises():
    from semseg_b200 import inference
    c = util.SW_CFG
    model = _model("psp", 7)
    p = inference.SlidingWindowPredictor(model, 7, 65, 65, c["mean"], c["std"], max_batch=8,
                                         anomaly=AnomalyScorer("sml"))
    with pytest.raises(ValueError):
        p(util.sw_image(seed=3, h=70, w=80), 80, [1.0])
    p.anomaly.statistics = (torch.zeros(5, dtype=torch.float64), torch.ones(5, dtype=torch.float64))
    with pytest.raises(ValueError):           # 5 classes of statistics, 7 of the predictor
        p(util.sw_image(seed=3, h=70, w=80), 80, [1.0])


# ------------------------------------------------------------------------------------------------ class moments
@pytest.mark.parametrize("shape,classes", [((1024, 2048), 19), ((97, 131), 150), ((3, 5), 4)])
def test_class_moments_match_oracle_and_are_deterministic(shape, classes):
    rng = np.random.default_rng(shape[1])
    pred = rng.integers(0, classes - 1, shape)              # class classes-1 never predicted
    ml = rng.standard_normal(shape) * 5 + 10 + pred
    p, m = torch.from_numpy(pred).cuda(), torch.from_numpy(ml).cuda()
    runs = []
    for _ in range(2):
        mom = torch.zeros((3, classes), dtype=torch.float64, device="cuda")
        ops.anomaly_class_moments(p, m, mom)
        runs.append(mom.cpu())
    assert torch.equal(runs[0], runs[1])
    ref = O.class_moments(pred, ml, classes)
    assert np.allclose(runs[0].numpy(), ref, rtol=1e-12, atol=0)
    assert runs[0][2, classes - 1] == 0
    mom = runs[0].clone().cuda()
    ops.anomaly_class_moments(p, m, mom)                    # adds into the caller's buffer
    assert np.allclose(mom.cpu().numpy(), 2 * ref, rtol=1e-12, atol=0)


# ------------------------------------------------------------------------------------------------ SML post-processing
def _blocky(rng, H, W, classes, block):
    coarse = rng.integers(0, classes, (H // block + 1, W // block + 1))
    return np.kron(coarse, np.ones((block, block), np.int64))[:H, :W]


@pytest.mark.parametrize("H,W,opts", [
    (256, 512, {}), (97, 131, dict(boundary_width=3, boundary_iterations=2, smooth_kernel=5, smooth_sigma=2.0,
                                   smooth_dilation=2)),
    (20, 30, {}),                                           # smaller than dilation * kernel
    (64, 48, dict(boundary_iterations=0)), (64, 48, dict(smooth_kernel=1)), (1, 77, dict(boundary_width=5)),
    (1024, 2048, {})])
def test_sml_matches_oracle_within_one_ulp(H, W, opts):
    classes = 6
    rng = np.random.default_rng(H + W)
    pred = _blocky(rng, H, W, 4, 9)                         # classes 4, 5 never predicted
    ml = rng.standard_normal((H, W)) * 2 + 8 + pred
    mean, std = O.class_statistics(pred, ml, classes)       # classes 4, 5 take the all-pixel statistics
    assert mean[4] == mean[5] == ml.mean()
    ref = O.sml_map(ml, pred, mean, std, **opts).astype(np.float32)
    sc = AnomalyScorer("sml", statistics=(mean, std), **opts)
    total = torch.zeros((classes + 2, H, W), dtype=torch.float64, device="cuda")
    total[classes] = torch.from_numpy(ml).cuda()
    got = sc.score_map(total, torch.from_numpy(pred).cuda()).cpu().numpy()
    err = np.abs(got.astype(np.float64) - ref.astype(np.float64))
    assert np.all(err <= np.spacing(np.abs(ref)).astype(np.float64) + 1e-13), float(err.max())
    again = sc.score_map(total, torch.from_numpy(pred).cuda()).cpu().numpy()
    assert np.array_equal(got, again)


# ------------------------------------------------------------------------------------------------ metrics
def _meter_case(rng, n, levels):
    vals = np.round(rng.standard_normal(levels), 3).astype(np.float32)
    s = rng.choice(vals, n)
    s[rng.random(n) < 0.03] = np.float32(-0.0)
    s[rng.random(n) < 0.03] = np.float32(0.0)
    y = (rng.random(n) < 0.05 + 0.4 * (s > 0.5)).astype(np.int64)
    y[rng.random(n) < 0.1] = 255
    return s, y


def test_meter_matches_oracle_over_several_updates():
    rng = np.random.default_rng(0)
    meter = AnomalyMeter()
    parts = [_meter_case(rng, n, lv) for n, lv in ((4_000_000, 50), (3_500_000, 2000), (2_700_000, 50),
                                                   (123_457, 7))]
    for k, (s, y) in enumerate(parts):
        lab = torch.from_numpy(y).cuda()
        meter.update(torch.from_numpy(s).cuda().view(-1, 1), (lab.to(torch.uint8) if k % 2 else lab).view(-1, 1))
    assert meter.count > 10_000_000
    got = meter.compute()
    s = np.concatenate([p[0] for p in parts])
    y = np.concatenate([p[1] for p in parts])
    auroc, ap, fpr95, pos, neg = O.metrics(s, y)
    assert (got["positives"], got["negatives"]) == (pos, neg)
    assert abs(got["auroc"] - auroc) <= 1e-12 and abs(got["ap"] - ap) <= 1e-12
    assert got["fpr95"] == fpr95
    assert meter.compute() == got                          # deterministic, and compute() keeps the pixels
    meter.reset()
    assert meter.count == 0


def test_meter_small_cases_match_sklearn_definition():
    from sklearn.metrics import average_precision_score, roc_auc_score
    rng = np.random.default_rng(1)
    for n, levels in ((10, 3), (1000, 1000), (4097, 5), (70_000, 2)):
        s, y = _meter_case(rng, n, levels)
        y[:2] = (0, 1)
        keep = y != 255
        meter = AnomalyMeter()
        meter.update(torch.from_numpy(s).cuda(), torch.from_numpy(y).cuda())
        got = meter.compute()
        assert abs(got["auroc"] - roc_auc_score(y[keep], s[keep])) <= 1e-12
        assert abs(got["ap"] - average_precision_score(y[keep], s[keep])) <= 1e-12
        assert got["fpr95"] == O.metrics(s, y)[2]


def test_meter_error_cases():
    def meter_of(s, y, ignore=255):
        m = AnomalyMeter(ignore)
        m.update(torch.tensor(s, dtype=torch.float32, device="cuda"), torch.tensor(y, device="cuda"))
        return m
    with pytest.raises(ValueError, match="label"):
        meter_of([0.1, 0.2, 0.3], [0, 1, 2]).compute()
    with pytest.raises(ValueError, match="non-finite"):
        meter_of([0.1, float("nan"), 0.3], [0, 1, 1]).compute()
    with pytest.raises(ValueError, match="non-finite"):
        meter_of([0.1, float("inf"), 0.3], [0, 1, 1]).compute()
    meter_of([0.1, float("nan"), 0.3, 0.2], [0, 255, 1, 1]).compute()    # void pixels may hold anything
    meter_of([0.1, 0.3, 0.2], [0, 7, 1], ignore=7).compute()
    with pytest.raises(ValueError, match="positives"):
        meter_of([0.1, 0.2], [0, 0]).compute()
    with pytest.raises(ValueError, match="positives"):
        meter_of([0.1, 0.2, 0.3], [1, 1, 255]).compute()
    m = AnomalyMeter()
    with pytest.raises(TypeError):
        m.update(torch.zeros(3, device="cuda"), torch.zeros(3, dtype=torch.int32, device="cuda"))
    with pytest.raises(ValueError):
        m.update(torch.zeros(3, device="cuda"), torch.zeros(4, dtype=torch.int64, device="cuda"))
    m.count = 2 ** 31 - 10                                  # as if 2^31 - 10 pixels were stored
    with pytest.raises(ValueError, match="2\\^31"):
        m.update(torch.zeros(11, device="cuda"), torch.zeros(11, dtype=torch.int64, device="cuda"))
    m.update(torch.zeros(9, device="cuda"), torch.zeros(9, dtype=torch.int64, device="cuda"))
    assert m.count == 2 ** 31 - 1
