"""CPU tier for the dense CRF (semseg_b200/densecrf.py, csrc/densecrf.cu): the float64 lattice contract
(tests/densecrf_oracle.py) agrees with the brute-force normalised Gaussian filter at the measured approximation error,
its mean-field labels agree with the brute-force CRF's, the CRF improves a synthetic case with displaced, blurred
boundaries in region accuracy and in the Boundary IoU counts, the module validates its arguments and has no CPU
fallback, and the entry points reject bad arguments before any CUDA call."""
import ctypes

import numpy as np
import pytest
import torch

from semseg_b200 import _lib
from semseg_b200.densecrf import DenseCRF
from tests import abl_oracle as A
from tests import densecrf_oracle as O

P = ctypes.c_void_p(16)      # never dereferenced: validation fails before any launch


def _err():
    return _lib.load().semseg_last_error()


# ------------------------------------------------------------------------------------------------ oracle
# Relative L2 error of the lattice filter against the brute force, measured on these 40 x 50 images (seeds 1 and 2):
# 0.9 % (d = 2, std 3), 1.7 % (std 1), 1.1 % (std 10); 2.0 % (d = 5, defaults), 2.4 % (xy 8), 2.2 % (xy 20, rgb 30).
# The gates leave a margin of about 1.5x; the approximation coarsens for small standard deviations (xy 3, rgb 5: 14 %).
@pytest.mark.parametrize("stds,gate", [((3.0,), 0.015), ((1.0,), 0.025), ((10.0,), 0.02),
                                       ((None, 80.0, 13.0), 0.03), ((None, 8.0, 13.0), 0.035),
                                       ((None, 20.0, 30.0), 0.035)])
@pytest.mark.parametrize("seed", [1, 2])
def test_lattice_oracle_approximates_the_brute_force_filter(stds, gate, seed):
    img, _, _ = O.synthetic_case(40, 50, 3, seed=seed)
    f = O.features(img, *stds)
    v = np.random.default_rng(seed).random((f.shape[0], 4))
    lat = O.Lattice(f)
    assert lat.V < f.shape[0] * (f.shape[1] + 1)
    got, ref = lat.filter(v), O.brute_filter(f, v)
    assert np.linalg.norm(got - ref) / np.linalg.norm(ref) < gate


def test_lattice_oracle_vertex_count_and_weights():
    img, _, _ = O.synthetic_case(40, 50, 3, seed=1)
    lat = O.Lattice(O.features(img, 3.0))
    assert lat.V == 291                                  # the float64 prototype's count at this size
    assert np.allclose(lat.weight.sum(1), 1.0) and (lat.weight > -1e-12).all()
    assert len(set(lat.keys)) == lat.V and all(len(k) == 2 for k in lat.keys)


@pytest.mark.parametrize("seed", [1, 2])
def test_meanfield_labels_agree_between_lattice_and_brute_force(seed):
    img, _, prob = O.synthetic_case(40, 50, 3, seed=seed)
    ql, qb = O.crf(img, prob), O.crf(img, prob, brute=True)
    assert (ql.argmax(1) != qb.argmax(1)).mean() <= 0.01      # measured: 0
    assert np.linalg.norm(ql - qb) / np.linalg.norm(qb) < 0.01


def test_oracle_crf_improves_displaced_boundaries():
    h, w, K = 40, 52, 3
    img, lab, prob = O.synthetic_case(h, w, K, shift=3, seed=4)
    before = prob.argmax(1).reshape(h, w)
    after = O.crf(img, prob).argmax(1).reshape(h, w)
    assert (after == lab).mean() > (before == lab).mean() + 0.1
    d = A.band_width(h, w)
    cb, ca = A.biou_counts(before[None], lab[None], K, 255, d), A.biou_counts(after[None], lab[None], K, 255, d)
    inter_b, union_b = cb[0].sum(), (cb[1] + cb[2] - cb[0]).sum()
    inter_a, union_a = ca[0].sum(), (ca[1] + ca[2] - ca[0]).sum()
    assert inter_a > inter_b and inter_a / union_a > inter_b / union_b + 0.3


def test_zero_iterations_is_the_clipped_softmax():
    prob = np.array([[0.0, 1.0], [0.3, 0.7]])
    q = O.meanfield(prob, [], [], 0, clip=1e-5)
    assert np.allclose(q[0], [1e-5 / (1 + 1e-5), 1 / (1 + 1e-5)]) and np.allclose(q[1], [0.3, 0.7])


# ------------------------------------------------------------------------------------------------ module
def test_constructor_defaults_and_repr():
    c = DenseCRF()
    assert (c.iterations, c.pos_weight, c.pos_xy_std, c.bi_weight, c.bi_xy_std, c.bi_rgb_std, c.clip) == \
        (5, 3.0, 3.0, 10.0, 80.0, 13.0, 1e-5)
    assert repr(c).startswith("DenseCRF(iterations=5, pos_weight=3")


@pytest.mark.parametrize("kw,bad,exc", [
    ("iterations", -1, ValueError), ("iterations", 2.5, TypeError), ("iterations", True, TypeError),
    ("pos_weight", -0.1, ValueError), ("bi_weight", float("nan"), ValueError), ("bi_weight", float("inf"), ValueError),
    ("pos_xy_std", 0.0, ValueError), ("bi_xy_std", -3.0, ValueError), ("bi_rgb_std", float("inf"), ValueError),
    ("bi_rgb_std", "13", TypeError), ("clip", 0.0, ValueError), ("clip", 1.0, ValueError), ("clip", -1e-5, ValueError),
    ("clip", 1e-39, ValueError), ("clip", 1e-45, ValueError),
])
def test_constructor_validation(kw, bad, exc):
    with pytest.raises(exc):
        DenseCRF(**{kw: bad})


def test_call_validation_and_no_cpu_fallback():
    crf = DenseCRF()
    img = np.zeros((4, 5, 3), np.float32)
    with pytest.raises(TypeError):
        crf(img, np.zeros((2, 4, 5), np.float32))
    with pytest.raises(TypeError):
        crf(img, torch.zeros((2, 4, 5), dtype=torch.float16))
    with pytest.raises(ValueError):
        crf(img, torch.zeros((4, 5)))
    with pytest.raises(_lib.SemsegError):
        crf(img, torch.zeros((2, 4, 5)))


def test_predictor_accepts_only_a_densecrf():
    from semseg_b200.inference import SlidingWindowPredictor
    net = torch.nn.Conv2d(3, 2, 1)
    with pytest.raises(TypeError):
        SlidingWindowPredictor(net, 2, 9, 9, [0, 0, 0], crf=object())
    assert SlidingWindowPredictor(net, 2, 9, 9, [0, 0, 0]).crf is None


# ------------------------------------------------------------------------------------------------ C-ABI validation
def _build(image=P, H=9, W=7, s=3.0, xy=80.0, rgb=13.0, lattice=P):
    return _lib.load().semseg_densecrf_build(image, H, W, s, xy, rgb, lattice, None)


def _meanfield(lattice=P, H=9, W=7, Vs=10, Va=20, prob=P, C=3, clip=1e-5, iterations=5, ws=3.0, wa=10.0, values=P, Q=P):
    return _lib.load().semseg_densecrf_meanfield(lattice, H, W, Vs, Va, prob, C, clip, iterations, ws, wa, values, Q,
                                                 None)


def _filter(lattice=P, H=9, W=7, Vs=10, Va=20, kernel=0, x=P, C=3, values=P, out=P):
    return _lib.load().semseg_densecrf_filter(lattice, H, W, Vs, Va, kernel, x, C, values, out, None)


def _keys(lattice=P, H=9, W=7, Vs=10, Va=20, kernel=0, s=3.0, xy=80.0, rgb=13.0, out=P):
    return _lib.load().semseg_densecrf_keys(lattice, H, W, Vs, Va, kernel, s, xy, rgb, out, None)


@pytest.mark.parametrize("call", [_build, _keys], ids=["build", "keys"])
def test_standard_deviations_and_key_overflow_are_rejected(call):
    for kw in ("s", "xy", "rgb"):
        for bad in (0.0, -1.0, float("nan"), float("inf")):
            assert call(**{kw: bad}) == -1 and b"standard deviations" in _err(), (kw, bad)
    assert call(H=2048, W=1024, xy=1e-3, rgb=1e-3) == -1 and b"more than 64" in _err()
    assert call(H=2048, W=1024, s=1e-9) == -1 and b"more than 64" in _err()
    assert call(H=0) == -1 and b"empty image" in _err()
    assert call(W=-3) == -1 and b"empty image" in _err()
    assert call(H=1 << 16, W=1 << 16) == -1 and b"too large" in _err()


@pytest.mark.parametrize("call", [_build, _keys], ids=["build", "keys"])
@pytest.mark.parametrize("kw", ["s", "xy", "rgb"])
@pytest.mark.parametrize("tiny", [1e-20, 1e-100, 1e-300, 5e-324])
def test_keys_beyond_exact_fp64_integers_are_rejected(call, kw, tiny):
    """Standard deviations so small that a coordinate range passes 2^52 (or the features overflow to inf) are rejected
    as key overflow, at every image size, before any integer conversion of the range."""
    for H, W in ((9, 7), (1, 2), (2, 1)):
        assert call(H=H, W=W, **{kw: tiny}) == -1 and b"more than 64" in _err(), (H, W)


def test_clip_at_the_fp32_limit():
    c = DenseCRF(clip=float(np.finfo(np.float32).tiny))
    assert c.clip == float(np.finfo(np.float32).tiny)
    for bad in (1e-39, 1e-45, 5e-324):
        assert _meanfield(clip=bad) == -1 and b"FLT_MIN" in _err(), bad
    assert _meanfield(clip=float(np.finfo(np.float32).tiny), Q=None) == -1 and b"null" in _err()


def test_build_rejects_null_pointers():
    for kw in ("image", "lattice"):
        assert _build(**{kw: None}) == -1 and b"null" in _err(), kw


def test_meanfield_rejects_bad_options():
    for bad in (-1, -100):
        assert _meanfield(iterations=bad) == -1 and b"iterations" in _err()
    for bad in (0.0, 1.0, -1e-5, 2.0, float("nan"), float("inf")):
        assert _meanfield(clip=bad) == -1 and b"clip" in _err(), bad
    for kw in ("ws", "wa"):
        for bad in (-0.5, float("nan"), float("inf"), float("-inf")):
            assert _meanfield(**{kw: bad}) == -1 and b"weights" in _err(), (kw, bad)
    assert _meanfield(H=0) == -1 and b"empty image" in _err()
    assert _meanfield(C=0) == -1 and b"C=0" in _err()
    for kw, bad in (("Vs", 0), ("Va", -1), ("Vs", 9 * 7 * 3 + 1), ("Va", 9 * 7 * 6 + 1)):
        assert _meanfield(**{kw: bad}) == -1 and b"vertex counts" in _err(), kw
    for kw in ("lattice", "prob", "values", "Q"):
        assert _meanfield(**{kw: None}) == -1 and b"null" in _err(), kw
    assert _meanfield(iterations=0, ws=0.0, wa=0.0, Q=None) == -1     # the options pass, the pointer does not


def test_filter_and_keys_reject_bad_arguments():
    for call in (_filter, _keys):
        assert call(kernel=2) == -1 and b"kernel 2" in _err()
        assert call(kernel=-1) == -1 and b"kernel -1" in _err()
        assert call(H=0) == -1 and b"empty image" in _err()
        assert call(Vs=0) == -1 and b"vertex counts" in _err()
        assert call(lattice=None) == -1 and b"null" in _err()
        assert call(out=None) == -1 and b"null" in _err()
    assert _filter(C=0) == -1 and b"C=0" in _err()
    for kw in ("x", "values"):
        assert _filter(**{kw: None}) == -1 and b"null" in _err(), kw


def test_workspace_sizes():
    lib = _lib.load()
    assert lib.semseg_densecrf_values_floats(9, 7, 10, 20, 3) == 2 * 30 * 3
    assert lib.semseg_densecrf_values_floats(9, 7, 0, 20, 3) == -1 and b"vertex counts" in _err()
    assert lib.semseg_densecrf_values_floats(9, 7, 10, 20, 0) == -1
    assert lib.semseg_densecrf_values_floats(0, 7, 10, 20, 3) == -1
    assert lib.semseg_densecrf_lattice_bytes(0, 5) == -1 and b"empty image" in _err()
    small = lib.semseg_densecrf_lattice_bytes(9, 7)
    assert 9 * 7 * 600 < small < 9 * 7 * 800 + 64 * 1024
    # the header's figure: about 700 bytes per pixel, 1.5 GB at 2048 x 1024
    big = lib.semseg_densecrf_lattice_bytes(1024, 2048)
    assert 1.3e9 < big < 1.6e9
    # worst-case values at 2048 x 1024 with 150 classes: V = N (d+1) for both kernels, 2 [V][C] buffers each
    n = 1024 * 2048
    assert 4 * lib.semseg_densecrf_values_floats(1024, 2048, 3 * n, 6 * n, 150) < 23e9
