"""Seeded psa_mask inputs shared by the tests that compare with the reference's own psa_mask kernels and by
tests/golden/make_psamask_digests.py, which stored those kernels' output digests."""
import numpy as np

CPU_CASES = [(2, 4, 5, 7, 9), (1, 6, 7, 5, 3), (2, 5, 5, 9, 9), (1, 30, 30, 59, 59), (1, 3, 9, 5, 17), (1, 1, 1, 1, 1)]
GPU_GEOMS = [(2, 30, 30, 59, 59), (1, 9, 12, 9, 7), (3, 5, 40, 9, 79), (1, 13, 13, 25, 25)]


def cpu_cases():
    """(key, psa_type, geometry, x, grad_out) in the order of the seed-11 stream."""
    rng = np.random.default_rng(11)
    for (n, h, w, mh, mw) in CPU_CASES:
        for t in (0, 1):
            x = rng.standard_normal((n, mh * mw, h, w)).astype(np.float32)
            g = rng.standard_normal((n, h * w, h, w)).astype(np.float32)
            yield "n%d_h%d_w%d_mh%d_mw%d_t%d" % (n, h, w, mh, mw, t), t, (n, h, w, mh, mw), x, g


def gpu_case(geom, psa_type):
    n, h, w, mh, mw = geom
    rng = np.random.default_rng(h * 31 + w + psa_type)
    x = rng.standard_normal((n, mh * mw, h, w)).astype(np.float32)
    g = rng.standard_normal((n, h * w, h, w)).astype(np.float32)
    return "n%d_h%d_w%d_mh%d_mw%d_t%d" % (n, h, w, mh, mw, psa_type), x, g


def gpu_cases():
    for geom in GPU_GEOMS:
        for t in (0, 1):
            key, x, g = gpu_case(geom, t)
            yield key, t, geom, x, g
