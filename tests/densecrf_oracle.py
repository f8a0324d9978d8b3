"""Float64 contract of the dense CRF (semseg_b200/densecrf.py, csrc/densecrf.cu).

Two filters feed one mean-field loop:
  * `brute_filter`: the exact symmetrically normalised Gaussian filter K~ v = n * K (n * v), n = (K 1 + 1e-20)^-1/2,
    summed over every pixel pair in row chunks (a few thousand pixels at most);
  * `Lattice`: an independent restatement of the permutohedral lattice of Adams, Baek & Davis (2010), as pydensecrf
    uses it: a Python dict keyed by coordinate tuples, filled in pixel order, [1 2 1] / 2 blur along each of the d+1
    lattice directions. The elevation, rounding and ranking are the same fp64 operations as the device build's, so the
    two find the same simplices and the same vertex set.
"""
import numpy as np


def features(image, pos_xy_std, bi_xy_std=None, bi_rgb_std=None):
    """[N, d] features of an H x W x 3 image (pixel i = y W + x): (x, y) / pos_xy_std when bi_xy_std is None (d = 2),
    else (x / bi_xy_std, y / bi_xy_std, rgb / bi_rgb_std) with the colour clamped to [0, 255] (d = 5)."""
    h, w = image.shape[:2]
    yy, xx = np.indices((h, w))
    if bi_xy_std is None:
        return np.stack([xx.ravel() / float(pos_xy_std), yy.ravel() / float(pos_xy_std)], 1)
    rgb = np.clip(np.asarray(image, np.float32).reshape(-1, 3), 0, 255).astype(np.float64) / float(bi_rgb_std)
    return np.concatenate([np.stack([xx.ravel() / float(bi_xy_std), yy.ravel() / float(bi_xy_std)], 1), rgb], 1)


def brute_filter(f, v, chunk=512):
    """Exact K~ v for features f [N, d] and values v [N, C]."""
    n_pix = f.shape[0]

    def apply(x):
        out = np.empty_like(x)
        sq = (f * f).sum(1)
        for a in range(0, n_pix, chunk):
            d2 = sq[a:a + chunk, None] + sq[None, :] - 2.0 * f[a:a + chunk] @ f.T
            out[a:a + chunk] = np.exp(-0.5 * np.maximum(d2, 0.0)) @ x
        return out
    norm = 1.0 / np.sqrt(apply(np.ones((n_pix, 1)))[:, 0] + 1e-20)
    return norm[:, None] * apply(norm[:, None] * v)


class Lattice:
    """Permutohedral lattice of features f [N, d]: vertex keys (d-tuples), per pixel its d+1 vertices and weights."""

    def __init__(self, f):
        f = np.asarray(f, np.float64)
        n_pix, d = f.shape
        self.d = d
        scale = np.array([np.sqrt(2.0 / 3.0) * (d + 1) / np.sqrt(float((i + 1) * (i + 2))) for i in range(d)])
        el = np.zeros((n_pix, d + 1))
        sm = np.zeros(n_pix)
        for j in range(d, 0, -1):
            cf = f[:, j - 1] * scale[j - 1]
            el[:, j] = sm - j * cf
            sm = sm + cf
        el[:, 0] = sm
        down = 1.0 / (d + 1)
        rd = np.floor(el * down + 0.5)
        rem0 = rd * (d + 1)
        total = rd.sum(1).astype(np.int64)
        rank = np.zeros((n_pix, d + 1), np.int64)
        for a in range(d):
            for b in range(a + 1, d + 1):
                less = (el[:, a] - rem0[:, a]) < (el[:, b] - rem0[:, b])
                rank[:, a] += less
                rank[:, b] += ~less
        for i in range(n_pix):
            s = total[i]
            if s > 0:
                hi = rank[i] >= d + 1 - s
                rem0[i, hi] -= d + 1
                rank[i] += np.where(hi, s - (d + 1), s)
            elif s < 0:
                lo = rank[i] < -s
                rem0[i, lo] += d + 1
                rank[i] += np.where(lo, d + 1 + s, s)
        bary = np.zeros((n_pix, d + 2))
        v = (el - rem0) * down
        for k in range(d + 1):
            np.add.at(bary, (np.arange(n_pix), d - rank[:, k]), v[:, k])
            np.add.at(bary, (np.arange(n_pix), d - rank[:, k] + 1), -v[:, k])
        bary[:, 0] += 1.0 + bary[:, d + 1]
        rem0 = rem0.astype(np.int64)
        index = {}
        self.vertex = np.zeros((n_pix, d + 1), np.int64)
        for i in range(n_pix):
            for r in range(d + 1):
                key = tuple(int(rem0[i, k] + (r if rank[i, k] <= d - r else r - (d + 1))) for k in range(d))
                self.vertex[i, r] = index.setdefault(key, len(index))
        self.weight = bary[:, :d + 1]
        self.keys = list(index)
        self.V = len(index)
        # blur neighbours along each direction j: key - 1 / + 1 with coordinate j moved by +d / -d
        self.nbr = np.full((d + 1, 2, self.V), -1, np.int64)
        for vid, key in enumerate(self.keys):
            for j in range(d + 1):
                n1 = tuple(key[k] + (d if k == j else -1) for k in range(d))
                n2 = tuple(key[k] + (-d if k == j else 1) for k in range(d))
                self.nbr[j, 0, vid] = index.get(n1, -1)
                self.nbr[j, 1, vid] = index.get(n2, -1)
        self.norm = 1.0 / np.sqrt(self.raw(np.ones((n_pix, 1)))[:, 0] + 1e-20)

    def raw(self, x):
        """Unnormalised lattice filter: splat, d+1 blur passes, slice."""
        C = x.shape[1]
        lat = np.zeros((self.V + 1, C))            # row V: the missing neighbour, kept at zero
        for r in range(self.d + 1):
            np.add.at(lat, self.vertex[:, r], self.weight[:, r:r + 1] * x)
        for j in range(self.d + 1):
            new = lat.copy()
            new[:self.V] = lat[:self.V] + 0.5 * (lat[self.nbr[j, 0]] + lat[self.nbr[j, 1]])
            new[self.V] = 0.0
            lat = new
        return (self.weight[:, :, None] * lat[self.vertex]).sum(1)

    def filter(self, x):
        return self.norm[:, None] * self.raw(self.norm[:, None] * x)


def softmax(z):
    z = z - z.max(1, keepdims=True)
    e = np.exp(z)
    return e / e.sum(1, keepdims=True)


def meanfield(prob, filters, weights, iterations, clip=1e-5):
    """Q [N, C] after `iterations` Potts mean-field updates; prob [N, C]; filters: callables [N, C] -> [N, C]."""
    logp = np.log(np.maximum(np.asarray(prob, np.float64), clip))
    Q = softmax(logp)
    for _ in range(iterations):
        Q = softmax(logp + sum(w * flt(Q) for flt, w in zip(filters, weights) if w > 0))
    return Q


def crf(image, prob, iterations=5, pos_weight=3.0, pos_xy_std=3.0, bi_weight=10.0, bi_xy_std=80.0, bi_rgb_std=13.0,
        clip=1e-5, brute=False):
    """The whole CRF of prob [N, C] (pixel-major) on an H x W x 3 image, lattice or brute-force filters."""
    fs = features(image, pos_xy_std)
    fa = features(image, None, bi_xy_std, bi_rgb_std)
    if brute:
        filters = [lambda q: brute_filter(fs, q), lambda q: brute_filter(fa, q)]
    else:
        ls, la = Lattice(fs), Lattice(fa)
        filters = [ls.filter, la.filter]
    return meanfield(prob, filters, [pos_weight, bi_weight], iterations, clip)


def synthetic_case(h=40, w=52, classes=3, shift=3, seed=0):
    """Piecewise-constant colour shapes with noise, their label map, and probabilities whose boundaries are displaced
    by `shift` pixels and blurred: (image float32 [h, w, 3], labels int64 [h, w], prob float64 [h*w, classes])."""
    rng = np.random.default_rng(seed)
    yy, xx = np.indices((h, w))
    lab = np.zeros((h, w), np.int64)
    lab[(yy - h * 0.45) ** 2 + (xx - w * 0.35) ** 2 < (0.28 * min(h, w)) ** 2] = 1
    lab[(xx > 0.6 * w) & (yy > 0.25 * h) & (yy < 0.8 * h)] = 2 % classes
    palette = np.array([[40, 60, 200], [220, 50, 40], [60, 200, 80]], np.float64)[:classes]
    image = np.clip(palette[lab] + rng.normal(0, 8, (h, w, 3)), 0, 255).astype(np.float32)
    moved = np.roll(np.roll(lab, shift, 0), shift, 1)
    onehot = np.eye(classes)[moved]
    from scipy import ndimage
    soft = np.stack([ndimage.uniform_filter(onehot[..., c], 2 * shift + 1, mode="nearest") for c in range(classes)], -1)
    prob = 0.15 / classes + 0.85 * soft
    prob /= prob.sum(-1, keepdims=True)
    return image, lab, prob.reshape(h * w, classes)
