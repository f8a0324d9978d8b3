"""GPU tier (-m gpu): the data-movement kernels of the training and eval path element by element at their window,
border and pitch edges: pyramid pooling (csrc/ppm.cu: ppm_pool, ppm_pool_bwd, ppm_upsample_concat, ppm_upsample_bwd),
bilinear resize (csrc/resize.cu), max-pool 3x3/s2 (csrc/pool.cu) and the layout kernels (csrc/layout.cu:
nchw_f32_to_nhwc_bf16, nhwc_bf16_to_nchw_f32, nhwc_f32_to_nchw_f32, space_to_phases, phases_to_space). Conventions as
in test_conv_edges_gpu.py and test_bn_edges_gpu.py, whose helpers are used here.

Reference. float64 on exactly what the kernel reads: the stored bf16 value, or hi + lo for split storage (exact in
fp32). The bilinear kernels compute scale = (in-1)/(out-1) (0 when out == 1), src = scale*dst, i0 = trunc(src) (clamped
to in-1 in resize.cu), i1 = min(i0+1, in-1), l1 = src - i0 and l0 = 1 - l1 in fp32, as ATen's fp32 path does; those are
reproduced in numpy float32, so each kernel is held to its own index and weight arithmetic, and only the combination is
done in float64. The adjoints weigh dy with the kernel's fp32 products wy*wx, wy = (i0 == i ? l0 : 0) + (i1 == i ? l1 : 0),
reproduced in float32 too. Every case is also cross-checked against float64 F.adaptive_avg_pool2d / F.interpolate /
F.max_pool2d(return_indices=True) (the max-pool on the CPU, where ATen's NaN rule was established) with a loose bound.
u = 2^-24.

Bounds (derived next to the kernel lines, see the functions below); the storage term is added to each: bf16, the stored
value is the round-to-nearest of some value within the bound; split, + 2^-16*|ref|:
  ppm_pool          acc += f per lane over ceil(npix/32) pixels, t += red[i] over the 32 lanes, t * fl(1/npix):
                    (ceil(npix/32) + 34)*u*sum|x|/npix;
  ppm_pool_bwd      acc = add, then one fmaf(d, fl(1/count), acc) per window holding the pixel:
                    (windows + 2)*u*(|add| + sum|d|/count);
  upsample / resize l0h*(l0w*v00 + l1w*v01) + l1h*(l0w*v10 + l1w*v11) with non-negative weights: 4u*sum w|v|; the
                    identity slice of ppm_upsample_concat is a copy and bit-exact in both planes;
  ppm_upsample_bwd  per lane one fmaf(wgt, d, acc) per pixel of a row with wy != 0, then the 32-lane sum:
                    (rows*ceil(W/32) + 32)*u*sum wgt|d|; cells no output pixel reaches are exactly 0;
  resize_bwd        one fmaf per output pixel with wgt != 0 (rows x columns of the candidate range): nnz*u*sum wgt|dy|;
  maxpool fwd       exact (hi + lo compared as a value: at a tie-to-even the planes may differ); argcode is ATen's index
                    mapped to the window position 0..8; bwd: at most 4 adds from 0: 3u*sum|dy|;
  layout            pure data movement: bit-exact against a torch restatement.

Teeth. Each case recomputes the reference without the contribution it guards (the windows past the 32nd of a pixel,
the overlap of non-divisible windows, the `add` term, the last 8-channel group, the border row and column, the l0/l1
assignment, the c_off slice, the shared top row of the max-pool windows) and asserts that the same bound flags at least
one element.

Every case also checks that a second call gives the same bits, that the inputs are unchanged, that a sentinel outside a
written channel slice survives, and mirrors the launch geometry (ppm_pool's grid (N*cells, ceil(C/64)); ew_blocks /
rs_blocks / mp_blocks: ceil(total/256) blocks capped at 16 per SM) to name the cases that run several grid-stride passes.
"""
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.test_bn_edges_gpu import SENTINEL, assert_outside_untouched, ew_grid
from tests.test_conv_edges_gpu import R_BF16, R_SPLIT, U, _act, cdiv, ratio, report, stored

pytestmark = pytest.mark.gpu

FORMS = [pytest.param(False, id="bf16"), pytest.param(True, id="x3")]


@pytest.fixture(scope="module", autouse=True)
def _device():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    yield


def _seed(name):
    return zlib.crc32(name.encode()) % 100000


def _L():
    from semseg_b200 import _lib as L
    return L


def act_ratio(out, ref, s, steps, split):
    return ratio(stored(out), ref, s, R_SPLIT if split else R_BF16, steps)


def act_in(n, h, w, c, split, gen, off=0, width=None):
    """(buffer, view): channels [off, off + c) of a random [N, H, W, width] activation."""
    width = width or c
    buf = _act(torch.randn((n, h, w, width), device="cuda", generator=gen), split)
    return buf, buf[..., off:off + c]


def act_out(n, h, w, width, split):
    from semseg_b200 import ops
    return ops.empty_act((n, h, w, width), split, "cuda").fill_(SENTINEL)


def passes(total, per_block=256):
    """Grid-stride passes of ew_blocks / rs_blocks / mp_blocks over `total` items of `per_block` per block."""
    return cdiv(total, ew_grid(total * 256 // per_block) * per_block)


# ------------------------------------------------------------------------------------------------ fp32 coordinates
def src_coords(n_out, n_in, clamp_i0):
    """(i0, i1, l0, l1) per output coordinate in the kernels' fp32 arithmetic (module docstring)."""
    s = np.float32(n_in - 1) / np.float32(n_out - 1) if n_out > 1 else np.float32(0)
    f = (s * np.arange(n_out, dtype=np.float32)).astype(np.float32)
    i0 = f.astype(np.int64)
    if clamp_i0:
        i0 = np.minimum(i0, n_in - 1)
    i1 = np.minimum(i0 + 1, n_in - 1)
    l1 = (f - i0.astype(np.float32)).astype(np.float32)
    l0 = (np.float32(1) - l1).astype(np.float32)
    return i0, i1, l0, l1


def interp_matrix(n_out, n_in, clamp_i0, swap=False):
    """[n_out, n_in] float64: the exact weights the forward combination applies (l0 at i0, l1 at i1, summed when they
    coincide). swap: l1 at i0 and l0 at i1 (teeth)."""
    i0, i1, l0, l1 = src_coords(n_out, n_in, clamp_i0)
    if swap:
        l0, l1 = l1, l0
    a = np.zeros((n_out, n_in))
    o = np.arange(n_out)
    np.add.at(a, (o, i0), l0.astype(np.float64))
    np.add.at(a, (o, i1), l1.astype(np.float64))
    return torch.from_numpy(a).cuda()


def adjoint_weights(n_out, n_in, clamp_i0):
    """[n_out, n_in] float32: wy = (i0 == i ? l0 : 0) + (i1 == i ? l1 : 0), the fp32 sum the backward kernels form."""
    i0, i1, l0, l1 = src_coords(n_out, n_in, clamp_i0)
    a = np.zeros((n_out, n_in), dtype=np.float32)
    o = np.arange(n_out)
    np.add.at(a, (o, i0), l0)
    np.add.at(a, (o, i1), l1)
    return torch.from_numpy(a).cuda()


def bilinear(v, ay, ax):
    """sum_ij ay[h, i] ax[w, j] v[n, i, j, c] in float64."""
    return torch.einsum("hi,wj,nijc->nhwc", ay, ax, v)


# ------------------------------------------------------------------------------------------------ PPM pool
def windows(length, b, rule="ceil"):
    """AdaptiveAvgPool2d's windows [floor(i*L/b), ceil((i+1)*L/b)); rule 'floor' ends at floor((i+1)*L/b) instead (the
    non-overlapping rule, teeth)."""
    return [((i * length) // b, -(-((i + 1) * length) // b) if rule == "ceil" else ((i + 1) * length) // b)
            for i in range(b)]


def max_windows(h, w, bins):
    cnt = torch.zeros((h, w), dtype=torch.int64)
    for b in bins:
        for hs, he in windows(h, b):
            for ws, we in windows(w, b):
                cnt[hs:he, ws:we] += 1
    return int(cnt.max())


# name: (N, H, W, C, bins, add, forward teeth, backward teeth)
PPM_POOL = {
    "psp50-60x60-c2048": (1, 60, 60, 2048, (1, 2, 3, 6), True, "group", "add"),
    "psp101-90x90-c72": (3, 90, 90, 72, (1, 2, 3, 6), True, "group", "group"),
    "9x12-c72": (3, 9, 12, 72, (1, 2, 3, 6), True, "overlap", "overlap"),
    "17x9-c8": (1, 17, 9, 8, (1, 2, 3, 6), True, "overlap", "overlap"),
    "6x6-c2048-exact": (3, 6, 6, 2048, (1, 2, 3, 6), True, "group", "add"),
    "5x7-c72": (1, 5, 7, 72, (1, 2, 3, 6), True, "overlap", "overlap"),
    "2x2-c8": (3, 2, 2, 8, (1, 2, 3, 6), True, "overlap", "overlap"),
    "1x3-c72": (1, 1, 3, 72, (1, 2, 3, 6), True, "overlap", "overlap"),
    "1x1-c8": (3, 1, 1, 8, (1, 2, 3, 6), True, "group", "cap32"),
    "1x1-c2048-noadd": (1, 1, 1, 2048, (1, 2, 3, 6), False, "group", "cap32"),
    "b1248-1x2-c72": (1, 1, 2, 72, (1, 2, 4, 8), True, "overlap", "cap32"),
    "b1248-2x2-c8": (3, 2, 2, 8, (1, 2, 4, 8), True, "overlap", "overlap"),
    "b2-16-2x2-c8": (1, 2, 2, 8, (2, 4, 8, 16), True, "overlap", "cap32"),
    "bins1-8-13x11-c72": (1, 13, 11, 72, (1, 2, 3, 4, 5, 6, 7, 8), True, "overlap", "overlap"),
    "one-bin6-9x12-c8-noadd": (3, 9, 12, 8, (6,), False, "overlap", "overlap"),
}


@pytest.mark.parametrize("split", FORMS)
@pytest.mark.parametrize("name", list(PPM_POOL))
def test_ppm_pool_and_bwd_element_bound(name, split):
    from semseg_b200 import ops
    L = _L()
    lib = L.load()
    n, h, w, c, bins, with_add, tf, tb = PPM_POOL[name]
    nb, cr = len(bins), 8
    gen = torch.Generator(device="cuda").manual_seed(_seed(name) + split)
    claims = ["N %d, %dx%d, C %d, bins %s" % (n, h, w, c, bins)]
    cells = sum(b * b for b in bins)
    claims.append("pool grid (%d, %d)%s" % (n * cells, cdiv(c, 64), ", partial 64-channel block" if c % 64 else ""))
    wmax = max_windows(h, w, bins)
    claims.append("up to %d windows per pixel" % wmax)
    if tb == "cap32":
        assert wmax > 32, "the case does not reach past 32 windows per pixel"
    if any(b > min(h, w) for b in bins):
        claims.append("bin larger than the map")
    bpass = cdiv(n * h * w, ew_grid(n * h * w * 32) * 8)
    claims.append("bwd %d grid-stride pass(es)" % bpass)
    if name.startswith("psp101"):
        assert bpass > 1

    # ---- forward, x a channel slice of a wider buffer
    xbuf, x = act_in(n, h, w, c, split, gen, 8, c + 16)
    x0 = xbuf.clone()
    pooled = [p.clone() for p in ops.ppm_pool(x, bins)]
    again = ops.ppm_pool(x, bins)
    assert all(torch.equal(a, b) for a, b in zip(pooled, again)), "not bit-identical on a second call"
    assert torch.equal(xbuf, x0)
    xs = stored(x)
    fw, ft, cross = 0.0, 0.0, 0.0
    for k, b in enumerate(bins):
        ref = torch.empty((n, b, b, c), device="cuda", dtype=torch.float64)
        s = torch.empty_like(ref)
        steps = torch.empty((1, b, b, 1), device="cuda", dtype=torch.float64)
        teeth = torch.zeros_like(ref)
        for ci, (hs, he) in enumerate(windows(h, b)):
            for cj, (ws, we) in enumerate(windows(w, b)):
                npix = (he - hs) * (we - ws)
                win = xs[:, hs:he, ws:we]
                ref[:, ci, cj] = win.sum((1, 2)) / npix
                s[:, ci, cj] = win.abs().sum((1, 2)) / npix
                steps[0, ci, cj, 0] = cdiv(npix, 32) + 34
        if tf == "overlap":
            for ci, (hs, he) in enumerate(windows(h, b, "floor")):
                for cj, (ws, we) in enumerate(windows(w, b, "floor")):
                    if he > hs and we > ws:
                        teeth[:, ci, cj] = xs[:, hs:he, ws:we].mean((1, 2))
        else:
            teeth = ref.clone()
            teeth[..., c - 8:] = 0
        fw = max(fw, act_ratio(pooled[k], ref, s, steps, split))
        ft = max(ft, act_ratio(pooled[k], teeth, s, steps, split))
        aten = F.adaptive_avg_pool2d(xs.permute(0, 3, 1, 2), b).permute(0, 2, 3, 1)
        cross = max(cross, float(((stored(pooled[k]) - aten).abs() / (s + 1e-30)).max()))
    assert cross < 2 ** -7, "ppm_pool vs F.adaptive_avg_pool2d: %.3g" % cross

    # ---- backward: add = dout[..., :C] of the (C + nb*Cr)-wide concat gradient, dx at pitch C + 16
    dpooled = [act_in(n, b, b, c, split, gen)[0] for b in bins]
    dbuf, add = act_in(n, h, w, c, split, gen, 0, c + nb * cr) if with_add else (None, None)
    ins = [d.clone() for d in dpooled] + ([dbuf.clone()] if with_add else [])
    dxbuf = act_out(n, h, w, c + 16, split)
    dx = dxbuf[..., 8:8 + c]
    barr, parr, larr, _ = ops._bin_args(bins, dpooled)
    outs = []
    for _ in range(2):
        L.check(lib.semseg_ppm_pool_bwd(parr, larr, barr, nb, n, h, w, c, ops._ptr(dx), ops._lo(dx), c + 16,
                                        ops._ptr(add), ops._lo(add), c + nb * cr if with_add else 0, ops._stream()),
                "semseg_ppm_pool_bwd")
        outs.append(dxbuf.clone())
    assert torch.equal(outs[0], outs[1]), "not bit-identical on a second call"
    assert all(torch.equal(a, b) for a, b in zip(ins, dpooled + ([dbuf] if with_add else [])))
    assert_outside_untouched(dxbuf, 8, c)
    assert torch.equal(ops.ppm_pool_bwd(dpooled, bins, n, h, w, c, add=add), dx), "ops wrapper differs"

    a64 = stored(add) if with_add else torch.zeros((n, h, w, c), device="cuda", dtype=torch.float64)
    ref, s = a64.clone(), a64.abs()
    teeth = torch.zeros_like(a64) if tb == "add" else a64.clone()
    cnt = torch.zeros((1, h, w, 1), device="cuda", dtype=torch.float64)
    for k, b in enumerate(bins):
        d = stored(dpooled[k])
        for ci, (hs, he) in enumerate(windows(h, b)):
            for cj, (ws, we) in enumerate(windows(w, b)):
                term = d[:, ci, cj, None, None, :] / ((he - hs) * (we - ws))
                ref[:, hs:he, ws:we] += term
                s[:, hs:he, ws:we] += term.abs()
                if tb == "cap32":    # the fixed 32-entry window list of the parent kernel
                    teeth[:, hs:he, ws:we] += term * (cnt[:, hs:he, ws:we] < 32)
                elif tb in ("add", "group"):
                    teeth[:, hs:he, ws:we] += term
                cnt[:, hs:he, ws:we] += 1
        if tb == "overlap":
            for ci, (hs, he) in enumerate(windows(h, b, "floor")):
                for cj, (ws, we) in enumerate(windows(w, b, "floor")):
                    if he > hs and we > ws:
                        teeth[:, hs:he, ws:we] += d[:, ci, cj, None, None, :] / ((he - hs) * (we - ws))
    if tb == "group":
        teeth[..., c - 8:] = 0
    assert int(cnt.max()) == wmax
    bw = act_ratio(dx, ref, s, cnt + 2, split)
    bt = act_ratio(dx, teeth, s, cnt + 2, split)
    claims.append("pool worst %.3g teeth %.3g (%s); bwd worst %.3g teeth %.3g (%s); vs ATen %.2g of mean|x|" %
                  (fw, ft, tf, bw, bt, tb, cross))
    report("ppm-pool-%s-%s" % (name, "x3" if split else "bf16"), claims, max(fw, bw), min(ft, bt))


# ------------------------------------------------------------------------------------------------ PPM upsample
# name: (N, H, W, C, Cr, bins, forward teeth, backward teeth)
PPM_UP = {
    "psp50-60x60-c2048-cr512": (1, 60, 60, 2048, 512, (1, 2, 3, 6), "border", "c_off"),
    "9x12-c8-cr72": (3, 9, 12, 8, 72, (1, 2, 3, 6), "group", "group"),
    "17x9-c2048-cr8": (1, 17, 9, 2048, 8, (1, 2, 3, 6), "swap", "border"),
    "1x7-c8-cr72": (1, 1, 7, 8, 72, (1, 2, 3, 6), "swap", "c_off"),
    "5x1-c8-cr8": (2, 5, 1, 8, 8, (1, 2, 3, 6), "swap", "border"),
    "1x1-c8-cr8": (1, 1, 1, 8, 8, (1, 2, 3, 6), "group", "c_off"),
    "b1-6x4-c8-cr8": (3, 6, 4, 8, 8, (1,), "group", "c_off"),
    "b6-on-2x2-c8-cr72": (3, 2, 2, 8, 72, (6,), "swap", "c_off"),
    "b3-6-on-4x5-c72-cr8": (1, 4, 5, 72, 8, (3, 6), "border", "border"),
}


@pytest.mark.parametrize("split", FORMS)
@pytest.mark.parametrize("name", list(PPM_UP))
def test_ppm_upsample_concat_and_bwd_element_bound(name, split):
    from semseg_b200 import ops
    L = _L()
    lib = L.load()
    n, h, w, c, cr, bins, tf, tb = PPM_UP[name]
    nb = len(bins)
    width = c + nb * cr
    gen = torch.Generator(device="cuda").manual_seed(_seed(name) + 7 + split)
    total = n * h * w * (c // 8 + nb * cr // 8)
    claims = ["N %d, %dx%d, C %d, Cr %d, bins %s" % (n, h, w, c, cr, bins),
              "concat %d grid-stride pass(es)" % passes(total)]
    if name.startswith("psp50"):
        assert passes(total) > 1
    if h == 1 or w == 1:
        claims.append("scale 0 along a unit dimension")
    if cr % 64:
        claims.append("partial 64-channel block in the backward")

    # ---- forward: x a slice (pitch C + 16), output pitch width + 8 (the last 8 channels keep the sentinel)
    xbuf, x = act_in(n, h, w, c, split, gen, 8, c + 16)
    feats = [act_in(n, b, b, cr, split, gen)[0] for b in bins]
    ins = [xbuf.clone()] + [f.clone() for f in feats]
    obuf = act_out(n, h, w, width + 8, split)
    out = obuf[..., :width]
    barr, parr, larr, _ = ops._bin_args(bins, feats)
    outs = []
    for _ in range(2):
        L.check(lib.semseg_ppm_upsample_concat(ops._ptr(x), ops._lo(x), c + 16, parr, larr, barr, nb, n, h, w, c, cr,
                                               ops._ptr(out), ops._lo(out), width + 8, ops._stream()),
                "semseg_ppm_upsample_concat")
        outs.append(obuf.clone())
    assert torch.equal(outs[0], outs[1]), "not bit-identical on a second call"
    assert all(torch.equal(a, b) for a, b in zip(ins, [xbuf] + feats))
    assert_outside_untouched(obuf, 0, width)
    assert torch.equal(out[..., :c], x), "the identity slice is not a bit-exact copy"
    assert torch.equal(ops.ppm_upsample_concat(x, feats, bins), out), "ops wrapper differs"
    fw, ft, cross = 0.0, 0.0, 0.0
    for k, b in enumerate(bins):
        v = stored(feats[k])
        ay, ax = interp_matrix(h, b, False), interp_matrix(w, b, False)
        ref = bilinear(v, ay, ax)
        s = bilinear(v.abs(), ay, ax)
        if tf == "swap":
            teeth = bilinear(v, interp_matrix(h, b, False, True), interp_matrix(w, b, False, True))
        elif tf == "border":
            teeth = ref.clone()
            teeth[:, -1] = ref[:, -2]
            teeth[:, :, -1] = ref[:, :, -2]
        else:
            teeth = ref.clone()
            teeth[..., cr - 8:] = 0
        got = out[..., c + k * cr:c + (k + 1) * cr]
        fw = max(fw, act_ratio(got, ref, s, 4, split))
        ft = max(ft, act_ratio(got, teeth, s, 4, split))
        aten = F.interpolate(v.permute(0, 3, 1, 2), size=(h, w), mode="bilinear", align_corners=True)
        cross = max(cross, float(((stored(got) - aten.permute(0, 2, 3, 1)).abs() / (s + 1e-30)).max()))
    assert cross < 2 ** -7, "ppm_upsample_concat vs F.interpolate: %.3g" % cross

    # ---- backward: dout the (C + nb*Cr)-wide concat gradient, c_off = C; dfeats prefilled with the sentinel
    dbuf, dout = act_in(n, h, w, width, split, gen)
    d0 = dbuf.clone()
    dfeats = [act_out(n, b, b, cr, split) for b in bins]
    barr, parr, larr, _ = ops._bin_args(bins, dfeats)
    outs = []
    for _ in range(2):
        L.check(lib.semseg_ppm_upsample_bwd(ops._ptr(dout), ops._lo(dout), width, c, parr, larr, barr, nb, n, h, w, cr,
                                            ops._stream()), "semseg_ppm_upsample_bwd")
        outs.append([f.clone() for f in dfeats])
    assert all(torch.equal(a, b) for a, b in zip(*outs)), "not bit-identical on a second call"
    assert torch.equal(dbuf, d0)
    assert all(torch.equal(a, b) for a, b in zip(ops.ppm_upsample_bwd(dout, c, bins, cr), dfeats)), "ops differs"
    bw, bt, unreached = 0.0, 0.0, 0
    dv = stored(dout).reshape(n, h * w, width)
    for k, b in enumerate(bins):
        wy, wx = adjoint_weights(h, b, False), adjoint_weights(w, b, False)
        wgt = (wy[:, None, :, None] * wx[None, :, None, :]).reshape(h * w, b * b).double()   # fp32 products
        d = dv[..., c + k * cr:c + (k + 1) * cr]
        ref = torch.einsum("pq,npc->nqc", wgt, d).reshape(n, b, b, cr)
        s = torch.einsum("pq,npc->nqc", wgt, d.abs()).reshape(n, b, b, cr)
        rows = (wy != 0).sum(0).double()                                   # rows with wy != 0, per ci
        steps = (rows * cdiv(w, 32) + 32)[None, :, None, None]
        if tb == "c_off":
            teeth = torch.einsum("pq,npc->nqc", wgt, dv[..., c - 8 + k * cr:c - 8 + (k + 1) * cr]).reshape(ref.shape)
        elif tb == "border":
            wgt_t = wgt.reshape(h, w, b * b).clone()
            wgt_t[-1] = 0
            wgt_t[:, -1] = 0
            teeth = torch.einsum("pq,npc->nqc", wgt_t.reshape(h * w, b * b), d).reshape(ref.shape)
        else:
            teeth = ref.clone()
            teeth[..., cr - 8:] = 0
        unreached += int((wgt.abs().sum(0) == 0).sum())
        bw = max(bw, act_ratio(dfeats[k], ref, s, steps, split))     # unreached cells: bound 0, must be exactly 0
        bt = max(bt, act_ratio(dfeats[k], teeth, s, steps, split))
    if name.startswith("b6-on-2x2"):
        assert unreached > 0
    claims.append("%d cells no output reaches (written 0)" % unreached)
    claims.append("fwd worst %.3g teeth %.3g (%s); bwd worst %.3g teeth %.3g (%s); vs ATen %.2g" %
                  (fw, ft, tf, bw, bt, tb, cross))
    report("ppm-up-%s-%s" % (name, "x3" if split else "bf16"), claims, max(fw, bw), min(ft, bt))


# ------------------------------------------------------------------------------------------------ bilinear resize
# name: (N, Hi, Wi, Ho, Wo, C, forward teeth, backward teeth)
RESIZE = {
    "psanet-59to30-c512": (1, 59, 59, 30, 30, 512, "border", "border"),
    "psanet-30to59-c512": (3, 30, 30, 59, 59, 512, "swap", "group"),
    "1to5x7-c8": (2, 1, 1, 5, 7, 8, "group", "group"),
    "6x9to1-c72": (1, 6, 9, 1, 1, 72, "swap", "group"),
    "1x1to1x1-c8": (3, 1, 1, 1, 1, 8, "group", "group"),
    "97to4-c72": (1, 97, 97, 4, 4, 72, "border", "border"),
    "4to97-c8": (1, 4, 4, 97, 97, 8, "swap", "border"),
    "13x7to5x11-c72": (2, 13, 7, 5, 11, 72, "swap", "border"),
}


@pytest.mark.parametrize("split", FORMS)
@pytest.mark.parametrize("name", list(RESIZE))
def test_resize_bilinear_fwd_bwd_element_bound(name, split):
    from semseg_b200 import ops
    L = _L()
    lib = L.load()
    n, hi, wi, ho, wo, c, tf, tb = RESIZE[name]
    gen = torch.Generator(device="cuda").manual_seed(_seed(name) + 11 + split)
    pf, pb = passes(n * ho * wo * c // 8), passes(n * hi * wi * c // 8)
    claims = ["N %d, %dx%d -> %dx%d, C %d" % (n, hi, wi, ho, wo, c), "grid-stride passes fwd %d bwd %d" % (pf, pb)]
    if name == "psanet-30to59-c512":
        assert pf > 1

    # ---- forward: x at pitch C + 16, y at pitch C + 8
    xbuf, x = act_in(n, hi, wi, c, split, gen, 8, c + 16)
    x0 = xbuf.clone()
    ybuf = act_out(n, ho, wo, c + 8, split)
    y = ybuf[..., :c]
    outs = []
    for _ in range(2):
        L.check(lib.semseg_resize_bilinear_fwd(ops._ptr(x), ops._lo(x), c + 16, n, hi, wi, c, ho, wo, ops._ptr(y),
                                               ops._lo(y), c + 8, ops._stream()), "semseg_resize_bilinear_fwd")
        outs.append(ybuf.clone())
    assert torch.equal(outs[0], outs[1]) and torch.equal(xbuf, x0)
    assert_outside_untouched(ybuf, 0, c)
    assert torch.equal(ops.resize_bilinear(x, (ho, wo)), y), "ops wrapper differs"
    v = stored(x)
    ay, ax = interp_matrix(ho, hi, True), interp_matrix(wo, wi, True)
    ref, s = bilinear(v, ay, ax), bilinear(v.abs(), ay, ax)
    if tf == "swap":
        teeth = bilinear(v, interp_matrix(ho, hi, True, True), interp_matrix(wo, wi, True, True))
    elif tf == "border":
        teeth = ref.clone()
        teeth[:, -1] = ref[:, -2]
        teeth[:, :, -1] = ref[:, :, -2]
    else:
        teeth = ref.clone()
        teeth[..., c - 8:] = 0
    fw, ft = act_ratio(y, ref, s, 4, split), act_ratio(y, teeth, s, 4, split)
    aten = F.interpolate(v.permute(0, 3, 1, 2), size=(ho, wo), mode="bilinear", align_corners=True).permute(0, 2, 3, 1)
    cross = float(((stored(y) - aten).abs() / (s + 1e-30)).max())
    assert cross < 2 ** -7, "resize_bilinear_fwd vs F.interpolate: %.3g" % cross

    # ---- backward: dy at pitch C + 16, dx at pitch C + 8
    dbuf, dy = act_in(n, ho, wo, c, split, gen, 8, c + 16)
    d0 = dbuf.clone()
    xgbuf = act_out(n, hi, wi, c + 8, split)
    dx = xgbuf[..., 8:]
    outs = []
    for _ in range(2):
        L.check(lib.semseg_resize_bilinear_bwd(ops._ptr(dy), ops._lo(dy), c + 16, n, hi, wi, c, ho, wo, ops._ptr(dx),
                                               ops._lo(dx), c + 8, ops._stream()), "semseg_resize_bilinear_bwd")
        outs.append(xgbuf.clone())
    assert torch.equal(outs[0], outs[1]) and torch.equal(dbuf, d0)
    assert_outside_untouched(xgbuf, 8, c)
    assert torch.equal(ops.resize_bilinear_bwd(dy, (hi, wi)), dx), "ops wrapper differs"
    wy, wx = adjoint_weights(ho, hi, True), adjoint_weights(wo, wi, True)
    wgt = (wy[:, None, :, None] * wx[None, :, None, :]).reshape(ho * wo, hi * wi).double()    # fp32 products
    g = stored(dy).reshape(n, ho * wo, c)
    ref = torch.einsum("pq,npc->nqc", wgt, g).reshape(n, hi, wi, c)
    s = torch.einsum("pq,npc->nqc", wgt, g.abs()).reshape(n, hi, wi, c)
    nnz = ((wy != 0).sum(0)[:, None] * (wx != 0).sum(0)[None, :]).double()[None, :, :, None]
    if tb == "border":
        wgt_t = wgt.reshape(ho, wo, hi * wi).clone()
        wgt_t[-1] = 0
        wgt_t[:, -1] = 0
        teeth = torch.einsum("pq,npc->nqc", wgt_t.reshape(ho * wo, hi * wi), g).reshape(ref.shape)
    else:
        teeth = ref.clone()
        teeth[..., c - 8:] = 0
    bw, bt = act_ratio(dx, ref, s, nnz, split), act_ratio(dx, teeth, s, nnz, split)
    # ATen's adjoint (autograd of F.interpolate) with the exact weights
    xr = torch.zeros((n, c, hi, wi), device="cuda", dtype=torch.float64, requires_grad=True)
    F.interpolate(xr, size=(ho, wo), mode="bilinear", align_corners=True).backward(stored(dy).permute(0, 3, 1, 2))
    bcross = float(((stored(dx) - xr.grad.permute(0, 2, 3, 1)).abs() / (s + 1e-30)).max())
    assert bcross < 2 ** -7, "resize_bilinear_bwd vs ATen's adjoint: %.3g" % bcross
    claims.append("chains up to %d fmaf" % int(nnz.max()))
    claims.append("fwd worst %.3g teeth %.3g (%s); bwd worst %.3g teeth %.3g (%s); vs ATen %.2g / %.2g" %
                  (fw, ft, tf, bw, bt, tb, cross, bcross))
    report("resize-%s-%s" % (name, "x3" if split else "bf16"), claims, max(fw, bw), min(ft, bt))


# ------------------------------------------------------------------------------------------------ max-pool
def _act_exact(v, split):
    """Activation of fp32 v whose stored value is bf16(v) (+ the lo plane bf16(v - hi) for finite v, 0 for +-inf and
    NaN, so an infinite input reads as infinite)."""
    hi = v.to(torch.bfloat16)
    if not split:
        return hi
    lo = torch.where(torch.isfinite(v), v - hi.float(), 0.0).to(torch.bfloat16)
    return torch.stack([hi, lo])


def maxpool_data(kind, n, h, w, c, gen):
    v = torch.randn((n, h, w, c), device="cuda", generator=gen)
    if kind == "relu":
        return v.clamp_min(0)
    if kind == "const":
        return torch.full_like(v, 1.5)
    if kind == "neginf":        # every window of the first half of the channels all -inf, the rest partly
        v[..., :c // 2] = -torch.inf
        v[..., c // 2:][v[..., c // 2:] < 0.5] = -torch.inf
        return v
    if kind == "inf":
        v[v > 1.0] = torch.inf
        v[v < -1.0] = -torch.inf
        return v
    if kind == "nan":
        # per channel residue: NaN at the first, the middle or the last tap of the window (1, 1) (rows and columns
        # 1..3), or two NaNs in it; plus scattered NaNs elsewhere
        r = torch.arange(c, device="cuda") % 4
        taps = {0: [(1, 1)], 1: [(2, 2)], 2: [(3, 3)], 3: [(1, 2), (3, 1)]}
        for q, pos in taps.items():
            for (a, b) in pos:
                if a < h and b < w:
                    v[:, a, b, r == q] = torch.nan
        v[torch.rand(v.shape, device="cuda", generator=gen) < 0.03] = torch.nan
        return v
    return v


def maxpool_ref(xs):
    """Window max and code in float64, ATen's rule: the first maximum in row-major window order, a NaN always taking
    over (so the last NaN), an all -inf window its first in-bounds tap."""
    n, h, w, c = xs.shape
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    pad = torch.full((n, 2 * ho + 1, 2 * wo + 1, c), torch.nan, device="cuda", dtype=torch.float64)
    ok = torch.zeros((2 * ho + 1, 2 * wo + 1), device="cuda", dtype=torch.bool)
    pad[:, 1:h + 1, 1:w + 1] = xs
    ok[1:h + 1, 1:w + 1] = True
    m = torch.full((n, ho, wo, c), -torch.inf, device="cuda", dtype=torch.float64)
    code = torch.full((n, ho, wo, c), 255, device="cuda", dtype=torch.int64)
    for t in range(9):
        kh, kw = divmod(t, 3)
        v = pad[:, kh:kh + 2 * ho:2, kw:kw + 2 * wo:2]
        valid = ok[kh:kh + 2 * ho:2, kw:kw + 2 * wo:2][None, :, :, None]
        upd = valid & ((v > m) | v.isnan() | (code == 255))
        m = torch.where(upd, v, m)
        code = torch.where(upd, t, code)
    return m, code


# name: (N, H, W, C, data)
MAXPOOL = {
    "1x1-c8": (2, 1, 1, 8, "randn"),
    "1x2-c64-relu": (1, 1, 2, 64, "relu"),
    "2x1-c72-relu": (1, 2, 1, 72, "relu"),
    "2x2-c8-relu": (3, 2, 2, 8, "relu"),
    "3x4-c128": (1, 3, 4, 128, "randn"),
    "4x3-c72-relu": (2, 4, 3, 72, "relu"),
    "5x4-c64-const": (1, 5, 4, 64, "const"),
    "5x5-c8-neginf": (1, 5, 5, 8, "neginf"),
    "4x5-c72-inf": (2, 4, 5, 72, "inf"),
    "5x5-c64-nan": (1, 5, 5, 64, "nan"),
    "4x4-c8-nan": (2, 4, 4, 8, "nan"),
    "237x237-c128-relu": (1, 237, 237, 128, "relu"),
    "237x236-c64-relu": (1, 237, 236, 64, "relu"),
}


@pytest.mark.parametrize("split", FORMS)
@pytest.mark.parametrize("name", list(MAXPOOL))
def test_maxpool3x3s2_exact_and_bwd_bound(name, split):
    from semseg_b200 import ops
    n, h, w, c, kind = MAXPOOL[name]
    gen = torch.Generator(device="cuda").manual_seed(_seed(name) + 13 + split)
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    claims = ["N %d, %dx%d -> %dx%d, C %d, %s" % (n, h, w, ho, wo, c, kind),
              "grid-stride passes fwd %d bwd %d" % (passes(n * ho * wo * c // 8), passes(n * h * w * c // 8))]
    x = _act_exact(maxpool_data(kind, n, h, w, c, gen), split)
    x0 = x.clone()
    y, code = ops.maxpool3x3s2_fwd(x)
    y2, code2 = ops.maxpool3x3s2_fwd(x)
    assert torch.equal(code, code2) and torch.equal(y.view(torch.int16), y2.view(torch.int16)), "not bit-identical"
    assert torch.equal(x.view(torch.int16), x0.view(torch.int16))
    xs = stored(x)
    m, mcode = maxpool_ref(xs)
    assert torch.equal(code.long(), mcode), "argcode differs from the window rule (%d elements)" % int(
        (code.long() != mcode).sum())
    hi = y[0] if split else y
    inf = m.isinf()
    # split storage keeps +-inf in the hi plane (act_st8's lo = bf16(inf - inf) is NaN): infinite maxima are compared
    # on hi, the rest as the value hi + lo
    got = torch.where(inf, hi.double(), stored(y))
    assert torch.equal(got.isnan(), m.isnan()), "NaN propagation differs"
    fin = ~m.isnan()
    assert torch.equal(got[fin], m[fin]), "max value not exact"
    # ATen on the CPU (NCHW float64): values and indices mapped to window positions
    av, ai = F.max_pool2d(xs.permute(0, 3, 1, 2).cpu(), 3, 2, 1, return_indices=True)
    av, ai = av.cuda().permute(0, 2, 3, 1), ai.cuda().permute(0, 2, 3, 1)
    oy = torch.arange(ho, device="cuda")[None, :, None, None]
    ox = torch.arange(wo, device="cuda")[None, None, :, None]
    acode = (ai // w - (2 * oy - 1)) * 3 + (ai % w - (2 * ox - 1))
    assert torch.equal(acode, mcode), "argcode differs from ATen's max_pool2d index (%d elements)" % int(
        (acode != mcode).sum())
    assert torch.equal(av.isnan(), m.isnan()) and torch.equal(av[fin], m[fin])
    nnan = int(m.isnan().sum())
    if kind == "nan":
        assert nnan > 0
        claims.append("%d NaN maxima" % nnan)
    if kind in ("relu", "const"):
        claims.append("%d tied inputs" % int((xs == xs.flatten()[0] if kind == "const" else xs == 0).sum()))

    # ---- backward: dy random, routed by argcode
    dy = _act_exact(torch.randn((n, ho, wo, c), device="cuda", generator=gen), split)
    dy0 = dy.clone()
    dx = ops.maxpool3x3s2_bwd(code, dy, (n, h, w, c))
    assert torch.equal(ops.maxpool3x3s2_bwd(code, dy, (n, h, w, c)), dx) and torch.equal(dy, dy0)
    assert torch.equal(code, code2)
    g = stored(dy)
    ref = torch.zeros((n, 2 * ho + 1, 2 * wo + 1, c), device="cuda", dtype=torch.float64)
    s, teeth, hits = torch.zeros_like(ref), torch.zeros_like(ref), torch.zeros_like(ref)
    for t in range(9):
        kh, kw = divmod(t, 3)
        sel = (mcode == t).double()
        sl = (slice(None), slice(kh, kh + 2 * ho, 2), slice(kw, kw + 2 * wo, 2))
        ref[sl] += g * sel
        s[sl] += g.abs() * sel
        hits[sl] += sel
        if kh > 0:                  # teeth: the top row of every window, where a pixel is shared with the window above
            teeth[sl] += g * sel
    crop = (slice(None), slice(1, h + 1), slice(1, w + 1))
    ref, s, teeth, hits = ref[crop], s[crop], teeth[crop], hits[crop]
    bw = act_ratio(dx, ref, s, 3, split)
    bt = act_ratio(dx, teeth, s, 3, split)
    hmax = int(hits.max())
    claims.append("a pixel receives from up to %d windows" % hmax)
    if h >= 3 and w >= 3 and kind in ("relu", "randn") and h * w > 100:
        assert hmax == 4, "no pixel shared by 4 windows took all four"
    claims.append("fwd exact, codes == ATen; bwd worst %.3g teeth %.3g (shared top row dropped)" % (bw, bt))
    if hmax < 2:                    # no shared pixel: the guard is the 1-window route itself
        bt = act_ratio(dx, torch.zeros_like(ref), s, 3, split)
    report("maxpool-%s-%s" % (name, "x3" if split else "bf16"), claims, bw, bt)


# ------------------------------------------------------------------------------------------------ layout
def _split_ref(v, split):
    hi = v.to(torch.bfloat16)
    return torch.stack([hi, (v - hi.float()).to(torch.bfloat16)]) if split else hi


@pytest.mark.parametrize("split", FORMS)
@pytest.mark.parametrize("c", [3, 8, 33, 64])
def test_nchw_nhwc_layout_bit_exact(c, split):
    """nchw_f32_to_nhwc_bf16 (pad channels zero, split lo = bf16_rn(v - bf16_rn(v))), nhwc_bf16_to_nchw_f32 on plain,
    split and channel-slice inputs, nhwc_f32_to_nchw_f32 at pitch > C; H*W = 153 is not a multiple of the 32-pixel
    tile, C = 33 not of the 32-channel one."""
    from semseg_b200 import ops
    n, h, w = 3, 17, 9
    gen = torch.Generator(device="cuda").manual_seed(c + split)
    x = torch.randn((n, c, h, w), device="cuda", generator=gen) * 3
    x0 = x.clone()
    a = ops.nchw_to_nhwc_bf16(x, pad_to=8, split=split)
    assert torch.equal(x, x0)
    cp = a.shape[-1]
    assert cp == -(-c // 8) * 8
    want = _split_ref(x.permute(0, 2, 3, 1).contiguous(), split)
    assert torch.equal(a[..., :c], want), "nchw_f32_to_nhwc_bf16"
    assert bool((a[..., c:] == 0).all()), "pad channels are not zero"
    assert torch.equal(ops.nchw_to_nhwc_bf16(x, pad_to=8, split=split), a), "not bit-identical on a second call"

    # back to NCHW: the stored fp32 value hi (+ lo), from a dense and from a channel-slice input
    back = ops.nhwc_bf16_to_nchw(a[..., :c])
    vals = (a[0].float() + a[1].float()) if split else a.float()
    assert torch.equal(back, vals[..., :c].permute(0, 3, 1, 2)), "nhwc_bf16_to_nchw_f32"
    buf = _act(torch.randn((n, h, w, c + 24), device="cuda", generator=gen), split)
    sl = buf[..., 8:8 + c]
    vals = (sl[0].float() + sl[1].float()) if split else sl.float()
    assert torch.equal(ops.nhwc_bf16_to_nchw(sl), vals.permute(0, 3, 1, 2)), "nhwc_bf16_to_nchw_f32 on a slice"

    f = torch.randn((n, h, w, c + 13), device="cuda", generator=gen)[..., 5:5 + c]
    assert f.stride(2) == c + 13
    assert torch.equal(ops.nhwc_f32_to_nchw(f), f.permute(0, 3, 1, 2)), "nhwc_f32_to_nchw_f32"
    print("\n[layout-c%d-%s] nchw->nhwc (pad %d->%d zero), nhwc->nchw plain / slice, f32 pitch %d: bit-exact" %
          (c, "x3" if split else "bf16", c, cp, c + 13))


@pytest.mark.parametrize("split", FORMS)
@pytest.mark.parametrize("n,h,w,c", [(1, 1, 1, 8), (2, 7, 9, 72), (1, 9, 4, 8), (3, 17, 13, 64), (1, 119, 119, 128)])
def test_space_phases_round_trip_bit_exact(n, h, w, c, split):
    """space_to_phases (x a channel slice, pitch > C) against xp[(ph*2+pw)*N + n, i, j] = x[n, 2i+ph, 2j+pw] (zero past
    the map), phases_to_space on its own against the same gather, and the round trip at odd H and W."""
    from semseg_b200 import ops
    gen = torch.Generator(device="cuda").manual_seed(n * h * w + c + split)
    buf = _act(torch.randn((n, h, w, c + 16), device="cuda", generator=gen), split)
    x = buf[..., 8:8 + c]
    b0 = buf.clone()
    xp = ops.space_to_phases(x)
    assert torch.equal(buf, b0)
    hh, wh = (h + 1) // 2, (w + 1) // 2
    want = torch.zeros_like(xp)
    for ph in range(2):
        for pw in range(2):
            q = ph * 2 + pw
            src = x[..., ph::2, pw::2, :]
            want[..., q * n:(q + 1) * n, :src.shape[-3], :src.shape[-2], :] = src
    assert torch.equal(xp, want), "space_to_phases"
    assert torch.equal(ops.space_to_phases(x), xp), "not bit-identical on a second call"
    assert torch.equal(ops.phases_to_space(xp, n, h, w), x), "round trip"

    zp = _act(torch.randn(tuple(xp.shape[-4:-1]) + (c,), device="cuda", generator=gen), split)
    z = ops.phases_to_space(zp, n, h, w)
    want = torch.empty_like(z)
    for ph in range(2):
        for pw in range(2):
            q = ph * 2 + pw
            dst = want[..., ph::2, pw::2, :]
            dst.copy_(zp[..., q * n:(q + 1) * n, :dst.shape[-3], :dst.shape[-2], :])
    assert torch.equal(z, want), "phases_to_space"
    print("\n[phases-%dx%dx%dx%d-%s] %d phase images of %dx%d, bit-exact both ways" %
          (n, h, w, c, "x3" if split else "bf16", 4 * n, hh, wh))
