"""GPU tier: Boundary IoU (metrics.boundaryIoUGPU, csrc/boundary.cu): the integer counts equal the contract's
(tests/abl_oracle.py) with ignored pixels, H != W, N > 1 and several band widths, and the paper's per-class cv2 form
on one case; `output` is left as it was and reruns give the same counts."""
import numpy as np
import pytest
import torch

from tests import abl_oracle as O
from tests.test_abl_cpu import _labels

pytestmark = pytest.mark.gpu


def _pair(shape, K, seed):
    t = _labels(*shape, classes=K, seed=seed)
    rng = np.random.default_rng(seed + 1)
    o = np.where(t == 255, rng.integers(0, K, shape), t)
    o = np.where(rng.random(shape) < 0.05, rng.integers(0, K, shape), np.roll(o, 1, axis=2))
    o[0, 0, :3] = K + 2                                        # out-of-range predictions are not counted
    return torch.from_numpy(o).cuda(), torch.from_numpy(t).cuda()


@pytest.mark.parametrize("shape,K,ratio", [((3, 41, 67), 5, 0.02), ((1, 64, 33), 19, 0.05), ((2, 97, 97), 150, 0.02),
                                           ((4, 7, 200), 3, 0.0)])
def test_counts_equal_the_oracle(shape, K, ratio):
    from semseg_b200.metrics import boundaryIoUGPU
    o, t = _pair(shape, K, seed=shape[1])
    o0 = o.clone()
    inter, union, target = boundaryIoUGPU(o, t, K, 255, dilation_ratio=ratio)
    assert torch.equal(o, o0)
    d = O.band_width(shape[1], shape[2], ratio)
    ref = O.biou_counts(o.cpu().numpy(), t.cpu().numpy(), K, 255, d)
    assert inter.dtype == torch.float32 and inter.shape == (K,)
    assert np.array_equal(inter.cpu().numpy(), ref[0])
    assert np.array_equal(target.cpu().numpy(), ref[2])
    assert np.array_equal(union.cpu().numpy(), ref[1] + ref[2] - ref[0])
    again = boundaryIoUGPU(o, t, K, 255, dilation_ratio=ratio)
    assert all(torch.equal(a, b) for a, b in zip((inter, union, target), again))


def test_counts_equal_the_papers_cv2_form():
    from semseg_b200.metrics import boundaryIoUGPU
    o, t = _pair((2, 45, 60), 4, seed=8)
    inter, union, target = boundaryIoUGPU(o, t, 4)
    ref = O.biou_counts_cv2(o.cpu().numpy(), t.cpu().numpy(), 4, 255, O.band_width(45, 60))
    assert np.array_equal(inter.cpu().numpy(), ref[0]) and np.array_equal(target.cpu().numpy(), ref[2])
    assert np.array_equal(union.cpu().numpy(), ref[1] + ref[2] - ref[0])
