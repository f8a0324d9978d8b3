"""GPU tier for the dense CRF (semseg_b200/densecrf.py, csrc/densecrf.cu) against the float64 contract of
tests/densecrf_oracle.py: the device lattice has the dict oracle's vertex count and key set; the normalised filter
equals the oracle lattice's to fp32 rounding over class counts, odd and one-pixel-wide images, and standard deviations
so large that the image falls into a handful of vertices or so small that no two pixels share one; the mean-field
marginals match after 0, 1 and 5 iterations; reruns are bit-identical; key overflow raises before any launch; the CRF
improves a synthetic boundary case in Boundary IoU; and SlidingWindowPredictor(crf=...) equals DenseCRF applied to the
predictor's own scores."""
import numpy as np
import pytest
import torch

from semseg_b200 import _lib, ops
from semseg_b200.densecrf import DenseCRF
from tests import densecrf_oracle as O
from tests import util

pytestmark = pytest.mark.gpu

DEFAULT = dict(pos_xy_std=3.0, bi_xy_std=80.0, bi_rgb_std=13.0)
HUGE = dict(pos_xy_std=1e4, bi_xy_std=1e4, bi_rgb_std=1e4)      # a handful of vertices
TINY = dict(pos_xy_std=0.05, bi_xy_std=0.2, bi_rgb_std=2.0)     # no two pixels share a vertex


def _image(h, w, seed):
    """Noisy colour regions (the CRF's use) with a band of uniform noise."""
    rng = np.random.default_rng(seed)
    yy, xx = np.indices((h, w))
    region = ((xx * 3 // max(w, 1)) + 2 * (yy * 2 // max(h, 1))) % 4
    palette = np.array([[30, 40, 200], [210, 60, 50], [70, 190, 90], [200, 200, 40]], np.float64)
    img = palette[region] + rng.normal(0, 10, (h, w, 3))
    img[h // 3:h // 3 + 2] = rng.random((min(2, h - h // 3), w, 3)) * 255
    return np.clip(img, 0, 255).astype(np.float32)


def _features(img, stds, kernel):
    return O.features(img, stds["pos_xy_std"]) if kernel == 0 else \
        O.features(img, None, stds["bi_xy_std"], stds["bi_rgb_std"])


def _build(img, stds):
    return ops.densecrf_build(torch.from_numpy(img).cuda(), stds["pos_xy_std"], stds["bi_xy_std"], stds["bi_rgb_std"])


# ------------------------------------------------------------------------------------------------ lattice
@pytest.mark.parametrize("shape,stds", [((40, 50), DEFAULT), ((17, 29), DEFAULT), ((1, 40), DEFAULT),
                                        ((40, 1), DEFAULT), ((23, 31), HUGE), ((20, 20), TINY),
                                        ((30, 37), dict(pos_xy_std=1.0, bi_xy_std=8.0, bi_rgb_std=5.0))])
def test_vertex_count_and_key_set_equal_the_dict_oracle(shape, stds):
    img = _image(*shape, seed=shape[0] + shape[1])
    lattice, V = _build(img, stds)
    for kernel in (0, 1):
        lat = O.Lattice(_features(img, stds, kernel))
        assert V[kernel] == lat.V, (kernel, V, lat.V)
        keys = ops.densecrf_keys(lattice, shape, V, kernel, **stds).cpu().numpy()
        assert keys.shape == (lat.V, lat.d)
        assert sorted(map(tuple, keys.tolist())) == sorted(lat.keys)
    if stds is TINY:
        assert V == (3 * img.shape[0] * img.shape[1], 6 * img.shape[0] * img.shape[1])
    if stds is HUGE:
        assert V[0] <= 8 and V[1] <= 32


# ------------------------------------------------------------------------------------------------ filter
# Observed worst case over these cases on an H100: 7.6e-7 relative L2 and 1.6e-6 of the largest value (appearance
# kernel, huge standard deviations); 1e-7 elsewhere. The gate is fp32 rounding with margin.
FILTER_GATE = 1e-5


@pytest.mark.parametrize("shape,stds,C", [((23, 31), DEFAULT, 1), ((23, 31), DEFAULT, 2), ((23, 31), DEFAULT, 19),
                                          ((23, 31), DEFAULT, 150), ((23, 31), DEFAULT, 256),
                                          ((17, 29), DEFAULT, 19), ((1, 40), DEFAULT, 5), ((40, 1), DEFAULT, 5),
                                          ((23, 31), HUGE, 19), ((20, 20), TINY, 19)])
def test_normalised_filter_equals_the_lattice_oracle(shape, stds, C):
    img = _image(*shape, seed=C)
    lattice, V = _build(img, stds)
    x = np.random.default_rng(C).random((shape[0] * shape[1], C))
    for kernel in (0, 1):
        ref = O.Lattice(_features(img, stds, kernel)).filter(x)
        got = ops.densecrf_filter(lattice, shape, V, kernel, torch.from_numpy(x).float().cuda()).double().cpu().numpy()
        rel = np.linalg.norm(got - ref) / np.linalg.norm(ref)
        assert rel < FILTER_GATE, (kernel, rel)
        assert np.abs(got - ref).max() <= 10 * FILTER_GATE * np.abs(ref).max(), kernel


# ------------------------------------------------------------------------------------------------ mean field
@pytest.mark.parametrize("iterations", [0, 1, 5])
@pytest.mark.parametrize("C", [3, 21])
def test_meanfield_matches_the_oracle(iterations, C):
    h, w = 36, 45
    img = _image(h, w, seed=7)
    logits = np.random.default_rng(C).normal(0, 2, (h * w, C))
    prob = O.softmax(logits)
    ref = O.crf(img, prob, iterations=iterations)
    crf = DenseCRF(iterations=iterations)
    got = crf(img, torch.from_numpy(prob.T.reshape(C, h, w)).cuda())
    assert got.shape == (C, h, w) and got.dtype == torch.float32
    got = got.double().cpu().numpy().reshape(C, -1).T
    assert np.abs(got - ref).max() < 2e-5          # observed on an H100: 2.6e-6 at 3 classes, 5 iterations
    top2 = np.sort(ref, 1)[:, -2:]
    clear = top2[:, 1] - top2[:, 0] > 1e-3
    assert clear.mean() > 0.95 and np.array_equal(got.argmax(1)[clear], ref.argmax(1)[clear])


def test_uint8_and_device_images_give_the_same_result():
    h, w, C = 24, 33, 4
    img = np.round(_image(h, w, seed=3)).astype(np.uint8)
    probs = torch.softmax(torch.randn((C, h, w), generator=torch.Generator().manual_seed(0)), 0).cuda()
    crf = DenseCRF()
    a = crf(img, probs)
    b = crf(img.astype(np.float32), probs.double())
    c = crf(torch.from_numpy(img).cuda(), probs)
    assert torch.equal(a, b) and torch.equal(a, c)


def test_reruns_are_bit_identical():
    h, w, C = 97, 131, 19
    img = _image(h, w, seed=5)
    probs = torch.softmax(torch.randn((C, h, w), generator=torch.Generator().manual_seed(1)), 0).cuda()
    crf = DenseCRF(iterations=5)
    a, b = crf(img, probs), crf(img, probs)
    assert torch.equal(a, b)
    l1, v1 = _build(img, DEFAULT)
    l2, v2 = _build(img, DEFAULT)
    assert v1 == v2
    for kernel in (0, 1):
        assert torch.equal(ops.densecrf_keys(l1, (h, w), v1, kernel, **DEFAULT),
                           ops.densecrf_keys(l2, (h, w), v2, kernel, **DEFAULT))


def test_key_overflow_raises_before_any_launch():
    img = torch.zeros((1024, 2048, 3), device="cuda")
    before = _lib.launch_count()
    with pytest.raises(_lib.SemsegError, match="more than 64"):
        ops.densecrf_build(img, 3.0, 1e-3, 1e-3)
    assert _lib.launch_count() == before


# ------------------------------------------------------------------------------------------------ boundaries
def test_crf_improves_a_synthetic_boundary_case_in_boundary_iou():
    from semseg_b200.metrics import boundaryIoUGPU, intersectionAndUnionGPU
    h, w, K = 40, 52, 3
    img, lab, prob = O.synthetic_case(h, w, K, shift=3, seed=4)
    probs = torch.from_numpy(prob.T.reshape(K, h, w)).cuda()
    refined = DenseCRF()(img, probs)
    target = torch.from_numpy(lab).cuda()[None]
    before, after = probs.argmax(0)[None], refined.argmax(0)[None]
    ib, ub, _ = boundaryIoUGPU(before, target, K)
    ia, ua, _ = boundaryIoUGPU(after, target, K)
    assert float(ia.sum()) > float(ib.sum()) and float((ia / ua).mean()) > float((ib / ub).mean()) + 0.3
    rb, _, tb = intersectionAndUnionGPU(before.clone(), target, K)
    ra, _, _ = intersectionAndUnionGPU(after.clone(), target, K)
    assert float(ra.sum()) > float(rb.sum()) + 0.1 * float(tb.sum())
    # the device CRF's labels are the oracle's
    ref = O.crf(img, prob).argmax(1).reshape(h, w)
    assert (after[0].cpu().numpy() == ref).mean() > 0.99


# ------------------------------------------------------------------------------------------------ predictor
@pytest.mark.parametrize("exact", [False, True])
def test_predictor_scores_are_densecrf_of_its_own_scores(exact):
    from semseg_b200 import inference
    c = util.SW_CFG
    classes, crop = 7, 65
    model = util.build_pspnet(50, classes=classes).cuda().eval()
    image = util.sw_image(seed=11, h=100, w=150)
    scales, base = [0.75, 1.0], 150
    crf = DenseCRF(iterations=3)
    plain = inference.SlidingWindowPredictor(model, classes, crop, crop, c["mean"], c["std"], max_batch=8)
    scores, _ = plain(image, base, scales, exact=exact)
    refined = inference.SlidingWindowPredictor(model, classes, crop, crop, c["mean"], c["std"], max_batch=8, crf=crf)
    got, amax = refined(image, base, scales, exact=exact)
    ref = crf(image, torch.from_numpy(scores).cuda().permute(2, 0, 1)).permute(1, 2, 0).double().cpu().numpy()
    assert got.dtype == np.float64 and got.shape == (100, 150, classes)
    assert np.array_equal(got, ref)
    assert np.array_equal(amax, got.argmax(2))
    none, amax2 = refined(image, base, scales, exact=exact, return_scores=False)
    assert (none is None) != exact and np.array_equal(amax2, amax)
