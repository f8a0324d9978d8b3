"""GPU tier (-m gpu): the tensor-core convolutions (csrc/conv_igemm.cu fprop / dgrad, csrc/conv_wgrad.cu, the K-slice
finish and wgrad_reduce) element by element at their tile, channel, tap and K-slice edges, and the classifier
(functional.conv_bias_f32) at real class counts.

Reference. float64 on exactly the operands the kernel reads: x / dy as stored (bf16, or the hi and lo planes
separately) and the weights unpacked from the packed slabs (wf / wd, hi and lo), not the fp32 masters. bf16:
sum x*w_hi. bf16x3: the kernel's three segments x_hi*w_hi + x_lo*w_hi + x_hi*w_lo (no lo*lo). What is left is fp32
accumulation and output rounding, so every element is held to

    |out - ref| <= r_out*|ref| + (c*L + e)*2^-24*S

  S      the same float64 convolution of |x| and |w| (for AFFINE: times |scale|, plus |shift| and |residual|);
  L      MMA steps in the longest accumulation chain feeding the element: K blocks per chain x 4 (K = 16 per step) x
         segments; for wgrad the pixel boxes per split x 4 x segments;
  e      round-to-nearest fp32 adds after the chain: the bias (1), the K-slice finish (k_slices), the split reduce
         (n_splits), the affine epilogue (3);
  r_out  2^-16 for hi/lo storage (16 mantissa bits), 2^-23 for fp32 outputs. For bf16 storage the rounding term
         r_out*|ref| (2^-8, bf16's unit roundoff) is replaced by its exact form: the stored value must be the
         round-to-nearest of some v with |v - ref| <= (c*L + e)*2^-24*S, i.e. |out - ref| minus half the gap above
         |out| is held to the accumulation term alone. Round to nearest spends its whole half-ulp on some element of
         every case, so a relative 2^-8*|ref| budget reads ~1 there and says nothing about the accumulation;
  c = 4  tools/probe_accum.py measures that the tensor core accumulates in fp32 with truncation, a bias towards zero
         of about 2^-24 per MMA step on average. Per step the worst case is one ulp (2^-23) lost when the step result
         is truncated plus one ulp lost when the addends are aligned to the largest exponent, each relative to a
         partial sum that is at most S: 2 * 2^-23 = 4 * 2^-24.

Teeth. Each case also recomputes the reference without the contribution the case exists to guard (one tap, the last
partial 64-channel K block, the last clipped pixel box, the last N tile, ...) and asserts that the same bound flags
at least one element, so the tolerance can see that bug class. No kernel is modified to show it.

Geometry. `choose_box`, `conv_block_n`, the K-slice count and wgrad's split choice are mirrored here and tied to the
library (semseg_conv_stats_rows, semseg_conv_k_slices, semseg_conv_wgrad_splits, semseg_conv_splitk_rows); each case
asserts the branch it names instead of assuming it. Every output is also checked to be bit-identical on a second call.
"""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
C_TRUNC = 4.0
R_BF16, R_SPLIT, R_F32 = "bf16", 2.0 ** -16, 2.0 ** -23   # R_BF16: round-to-nearest bf16 storage
X3_MAX_KBLOCKS = 8


@pytest.fixture(scope="module", autouse=True)
def _device():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def cdiv(a, b):
    return -(-a // b)


# ------------------------------------------------------------------------------------------------ geometry mirror
def choose_box(h, w, max_pixels):
    """csrc/host_common.cu::choose_box."""
    best, bb = -1.0, (1, 1)
    for bw in range(1, min(w, max_pixels) + 1):
        bh = min(max_pixels // bw, h, 256)
        if bh < 1:
            continue
        th = cdiv(h, bh)
        bh = cdiv(h, th)
        util = h * w / (th * cdiv(w, bw) * max_pixels)
        if util > best + 1e-9 or (util > best - 1e-9 and bw > bb[1]):
            best, bb = util, (bh, bw)
    return bb


def conv_block_n(cout):
    """csrc/conv_igemm.cu::conv_block_n."""
    if cout % 256 == 0 or cout > 128:
        return 256
    return 128 if cout > 64 else 64


def fprop_geom(n, h, w, cin, cout, taps, k_slices=1):
    g = dict(n=n, h=h, w=w, cin=cin, cout=cout, taps=taps)
    g["bh"], g["bw"] = choose_box(h, w, 128)
    g["tiles"] = n * cdiv(h, g["bh"]) * cdiv(w, g["bw"])
    g["block_n"] = conv_block_n(cout)
    g["n_tiles"] = cdiv(cout, g["block_n"])
    g["kblocks"] = taps * cdiv(cin, 64)
    g["kb_per_slice"] = cdiv(g["kblocks"], k_slices)
    g["k_slices"] = cdiv(g["kblocks"], g["kb_per_slice"])
    g["items"] = g["tiles"] * g["n_tiles"] * g["k_slices"]
    g["grid"] = min(g["items"], _sms())
    return g


def stat_masks(g):
    """Valid-row masks of every (pixel box, 32-row statistics warp), as the epilogue's ballot computes them."""
    bh, bw, th, tw = g["bh"], g["bw"], cdiv(g["h"], g["bh"]), cdiv(g["w"], g["bw"])
    masks = []
    for ty in range(th):
        for tx in range(tw):
            h0, w0 = ty * bh, tx * bw
            for wq in range(4):
                m = 0
                for lane in range(32):
                    r = wq * 32 + lane
                    if r < bh * bw and h0 + r // bw < g["h"] and w0 + r % bw < g["w"]:
                        m |= 1 << lane
                masks.append(m)
    return masks


def non_prefix_mask(g):
    return any(m & (m + 1) for m in stat_masks(g))


def wgrad_geom(n, h, w, cin, cout, taps, split, n_splits=0):
    """csrc/conv_wgrad.cu::wgrad_geometry."""
    g = dict(n=n, h=h, w=w, cin=cin, cout=cout, taps=taps)
    bh, bw = choose_box(h, w, 64)
    g["boxes"] = n * cdiv(h, bh) * cdiv(w, bw)
    g["co_tiles"] = cdiv(cout, 128)
    block_n = 256 if cin > 128 else (128 if cin > 64 else 64)
    ci_tiles, tu, unit_taps = cdiv(cin, block_n), 1, taps
    if taps > 1 and cin <= 128:
        tu = 4 // cdiv(cin, 64)
        unit_taps, block_n, ci_tiles = cdiv(taps, tu), 256, 1
    g.update(block_n=block_n, ci_tiles=ci_tiles, tu=tu, unit_taps=unit_taps)
    g["unit_sizes"] = [min(tu, taps - u * tu) for u in range(unit_taps)]
    units = unit_taps * g["co_tiles"] * ci_tiles
    splits = n_splits
    if splits <= 0:
        slots, boxes = _sms(), g["boxes"]
        max_s = min(max(boxes // 16, 1), 64)
        best, splits = -1.0, 1
        for sp in range(1, max_s + 1):
            waves = units * sp / slots
            kb = boxes / sp
            score = (waves / math.ceil(waves)) * (kb / (kb + 8.0)) * (1.0 if waves >= 1.0 else waves)
            if score > best + 1e-9:
                best, splits = score, sp
        if split:
            splits = max(splits, cdiv(boxes, 21))
    g["boxes_per_split"] = cdiv(g["boxes"], splits)
    g["n_splits"] = cdiv(g["boxes"], g["boxes_per_split"])
    return g


def splitk_chunk_rows(m):
    """csrc/bn.cu::splitk_chunk_rows."""
    rows = max(cdiv(m, 2048), 128)
    return (rows + 31) & ~31


# ------------------------------------------------------------------------------------------------ float64 reference
def _shift(x, dh, dw, img_add, out_nhw):
    """out[n, h, w] = x[n + img_add, h + dh, w + dw], zero outside x (the TMA halo fill)."""
    n_out, h_out, w_out = out_nhw
    nin, hin, win = x.shape[:3]
    out = x.new_zeros((n_out, h_out, w_out, x.shape[3]))
    n0, n1 = max(0, -img_add), min(n_out, nin - img_add)
    h0, h1 = max(0, -dh), min(h_out, hin - dh)
    w0, w1 = max(0, -dw), min(w_out, win - dw)
    if n0 < n1 and h0 < h1 and w0 < w1:
        out[n0:n1, h0:h1, w0:w1] = x[n0 + img_add:n1 + img_add, h0 + dh:h1 + dh, w0 + dw:w1 + dw]
    return out


def tap_conv(x, slab, taps, cout, img_add=None, out_nhw=None):
    """sum_t shift(x, t) @ slab[wtap(t)][:cout, :Cin]^T in float64."""
    out_nhw = out_nhw or tuple(x.shape[:3])
    cin = x.shape[3]
    acc = None
    for i, (dh, dw, wt) in enumerate(taps):
        xs = _shift(x, dh, dw, img_add[i] if img_add else 0, out_nhw)
        t = xs @ slab[wt, :cout, :cin].t()
        acc = t if acc is None else acc + t
    return acc


def planes(t, split):
    """float64 planes of an activation or packed slab as the kernel reads them: [hi] or [hi, lo]."""
    return [t[0].double(), t[1].double()] if split else [t.double()]


def _segments(x_planes, w_planes):
    if len(x_planes) == 1:
        return [(x_planes[0], w_planes[0])]
    (xh, xl), (wh, wl) = x_planes, w_planes
    return [(xh, wh), (xl, wh), (xh, wl)]


def seg_conv(x_planes, w_planes, taps, cout, img_add=None, out_nhw=None):
    """(ref, S): the kernel's segments summed, and the same with |x|, |w|."""
    ref = s = 0
    for xa, wa in _segments(x_planes, w_planes):
        ref = ref + tap_conv(xa, wa, taps, cout, img_add, out_nhw)
        s = s + tap_conv(xa.abs(), wa.abs(), taps, cout, img_add, out_nhw)
    return ref, s


def stored(t):
    """float64 value of a stored activation (hi + lo for split storage) or fp32 tensor."""
    if t.dtype == torch.float32:
        return t.double()
    return t[0].double() + t[1].double() if t.dim() == 5 else t.double()


def ratio(out, ref, s, r_out, steps):
    """max |out - ref| / bound; a zero bound admits only an exact zero difference. r_out = R_BF16: out is stored in bf16,
    so the half gap above |out| (2^(floor(log2|out|) - 8)) is taken off the error before it meets the accumulation
    term."""
    err = (out - ref).abs()
    if r_out == R_BF16:
        # floor(log2|out|) = frexp exponent - 1, exactly (a device log2 may land just below the integer at 2^k)
        half = torch.where(out != 0, torch.ldexp(torch.ones_like(out), torch.frexp(out)[1] - 9), 0.0)
        err = (err - half).clamp_min(0.0)
        bound = steps * U * s
    else:
        bound = r_out * ref.abs() + steps * U * s
    r = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))
    return float(r.max())


def report(name, claims, worst, teeth):
    print("\n[%s] %s | worst |err|/bound %.3g | teeth %.3g" % (name, "; ".join(claims), worst, teeth))
    assert worst <= 1.0, "%s: an element exceeds the bound (worst ratio %.3g)" % (name, worst)
    assert teeth > 1.0, "%s: the bound cannot see the guarded contribution (teeth ratio %.3g)" % (name, teeth)


def _act(t, split):
    """fp32 NHWC -> activation as the network stores it (bf16, or hi/lo planes)."""
    from semseg_b200 import ops
    return ops.f32_to_act(t.contiguous(), split) if split else t.to(torch.bfloat16)


# ------------------------------------------------------------------------------------------------ fprop / dgrad
# id: (N, H, W, Cin, Cout, k, dilation, options). options: epi (raw / affine / f32), stats, dgrad (run the transposed
# taps on the wd slab), xslice (channel offset of x inside a buffer 2*Cin + 16 wide), res (residual: channel offset,
# buffer width), nulls (AFFINE without scale / shift), oslice (F32 output: channel offset, buffer width), forms,
# teeth (what the reference drops).
FPROP = {
    # pixel grid
    "grid-exact-8x16": (2, 8, 16, 64, 64, 3, 1, dict(stats=True, teeth="tap")),
    "grid-3x5-below-one-box": (2, 3, 5, 64, 128, 3, 1, dict(stats=True, teeth="tap")),
    "grid-h1-w300": (1, 1, 300, 64, 64, 3, 1, dict(stats=True, teeth="box")),
    "grid-h300-w1": (1, 300, 1, 64, 64, 3, 1, dict(stats=True, teeth="box")),
    "grid-61x67-clipped": (1, 61, 67, 64, 64, 3, 1, dict(stats=True, teeth="box")),
    "grid-61x67-clipped-1x1": (1, 61, 67, 64, 64, 1, 1, dict(stats=True, teeth="box")),
    "grid-n16-multi-item": (16, 27, 27, 64, 320, 1, 1, dict(stats=True, teeth="box")),
    # output channels
    "cout64-affine-res": (1, 13, 11, 64, 64, 3, 1, dict(epi="affine", res=(0, 64), teeth="tap")),
    "cout128-raw": (1, 13, 11, 64, 128, 3, 2, dict(stats=True, teeth="tap")),
    "cout192-affine": (1, 9, 11, 128, 192, 3, 1, dict(epi="affine", res=(64, 320), teeth="ntile")),
    "cout320-raw-two-ntiles": (2, 9, 11, 128, 320, 1, 1, dict(stats=True, teeth="ntile")),
    "cout2048-affine": (1, 6, 7, 512, 2048, 1, 1, dict(epi="affine", res=(0, 2048), teeth="ntile")),
    "f32-19-odd-pitch": (2, 7, 9, 512, 19, 1, 1, dict(epi="f32", teeth="lastch")),
    "f32-21-slice-odd-offset": (2, 7, 9, 512, 21, 1, 1, dict(epi="f32", oslice=(3, 40), teeth="lastch")),
    "f32-150": (2, 7, 9, 512, 150, 1, 1, dict(epi="f32", teeth="ntile")),
    "f32-152-slice": (2, 7, 9, 512, 152, 1, 1, dict(epi="f32", oslice=(8, 168), teeth="ntile")),
    # input channels
    "cin8": (2, 10, 12, 8, 64, 3, 1, dict(stats=True, teeth="kblock")),
    "cin24-dgrad-of-cls": (2, 10, 12, 24, 512, 1, 1, dict(dgrad=True, teeth="kblock")),
    "cin32-xslice-low": (2, 10, 12, 32, 64, 3, 1, dict(xslice=0, teeth="kblock")),
    "cin72-xslice-high": (2, 10, 12, 72, 128, 3, 1, dict(xslice=72, teeth="kblock")),
    "cin152-dgrad-of-cls": (2, 10, 12, 152, 512, 1, 1, dict(dgrad=True, xslice=152, teeth="kblock")),
    "cin4096": (1, 5, 7, 4096, 128, 1, 1, dict(epi="affine", teeth="kblock")),
    "affine-null-scale-shift": (1, 9, 10, 128, 128, 3, 1, dict(epi="affine", nulls=True, res=(8, 144), teeth="res")),
    # taps
    "1x1": (2, 9, 9, 64, 64, 1, 1, dict(teeth="kblock")),
    "3x3-d1-dgrad": (2, 9, 11, 128, 64, 3, 1, dict(dgrad=True, teeth="tap")),
    "3x3-d2": (1, 17, 15, 64, 64, 3, 2, dict(teeth="tap")),
    "3x3-d2-dgrad": (1, 17, 15, 64, 64, 3, 2, dict(dgrad=True, teeth="tap")),
    "3x3-d4-on-9x9": (2, 9, 9, 512, 512, 3, 4, dict(stats=True, teeth="tap")),
    "3x3-d4-dgrad": (2, 9, 9, 512, 512, 3, 4, dict(dgrad=True, teeth="tap")),
    "3x3-d12-all-halo": (1, 12, 11, 64, 64, 3, 12, dict(stats=True, teeth="halo")),
    "3x3-d12-all-halo-dgrad": (1, 7, 12, 64, 64, 3, 12, dict(dgrad=True, teeth="halo")),
    # K slicing (bf16x3): 8, 9, 18 and 576 K blocks, RAW + statistics and AFFINE + residual + ReLU finishes
    "kslice-8-raw": (2, 7, 9, 512, 64, 1, 1, dict(stats=True, forms=(True,), teeth="kblock")),
    "kslice-9-raw": (2, 7, 9, 64, 64, 3, 1, dict(stats=True, forms=(True,), teeth="tap")),
    "kslice-9-affine": (2, 7, 9, 64, 128, 3, 1, dict(epi="affine", res=(0, 128), forms=(True,), teeth="tap")),
    "kslice-18-raw": (2, 7, 9, 128, 64, 3, 2, dict(stats=True, forms=(True,), teeth="tap")),
    "kslice-576-cls-raw": (1, 6, 7, 4096, 512, 3, 1, dict(stats=True, forms=(True,), teeth="kblock")),
    "kslice-576-cls-affine": (1, 6, 7, 4096, 512, 3, 1, dict(epi="affine", res=(0, 512), forms=(True,),
                                                              teeth="kblock")),
}

FPROP_PARAMS = [pytest.param(name, split, id="%s-%s" % (name, "x3" if split else "bf16"))
                for name, case in FPROP.items() for split in case[7].get("forms", (False, True))]


def _stats_ratio(sp, y64, depth):
    """float64 merge of the statistics rows vs float64 sum and sum of squares of the stored outputs y64 [M, C]: worst
    |err| / bound, with fp32 sums of at most `depth` terms per row (+1 rounding of the square)."""
    sp = sp.double()
    rs = ((sp[:, 0].sum(0) - y64.sum(0)).abs() / (depth * U * y64.abs().sum(0)).clamp_min(1e-300)).max()
    rq = ((sp[:, 1].sum(0) - (y64 * y64).sum(0)).abs() / ((depth + 1) * U * (y64 * y64).sum(0)).clamp_min(1e-300)).max()
    return max(float(rs), float(rq))


@pytest.mark.parametrize("name,split", FPROP_PARAMS)
def test_conv_fprop_element_bound(name, split):
    from semseg_b200 import ops, _lib
    n, h, w, cin, cout, k, dil, o = FPROP[name]
    epi = {"raw": ops.EPI_RAW, "affine": ops.EPI_AFFINE, "f32": ops.EPI_F32}[o.get("epi", "raw")]
    g = torch.Generator(device="cuda").manual_seed(hash(name) % 10007)
    dev = "cuda"
    nseg = 3 if split else 1
    claims = []

    # operands: x (optionally a channel slice of a wider buffer whose other channels are non-zero), packed weights
    xoff = o.get("xslice")
    width = cin if xoff is None else 2 * cin + 16
    xbuf = _act(torch.randn((n, h, w, width), device=dev, generator=g), split)
    x = xbuf[..., xoff:xoff + cin] if xoff is not None else xbuf
    if xoff is not None:
        assert ops._nhwc_meta(x)[4] > cin
        claims.append("x is channels [%d, %d) of a %d-channel buffer (pitch > Cin)" % (xoff, xoff + cin, width))
    if o.get("dgrad"):
        wt = torch.randn((cin, cout, k, k), device=dev, generator=g) / (cin * k * k) ** 0.5   # dgrad: Cin of the run
        pw = ops.pack_weights(wt, split=split)
        slab, taps = pw.wd, ops.conv_taps(k, dil, transpose=True)
        claims.append("dgrad: transposed taps on the wd slab")
    else:
        wt = torch.randn((cout, cin, k, k), device=dev, generator=g) / (cin * k * k) ** 0.5
        pw = ops.pack_weights(wt, split=split)
        slab, taps = pw.wf, ops.conv_taps(k, dil)
    kw = {}
    scale = shift = res = None
    if epi == ops.EPI_AFFINE:
        if not o.get("nulls"):
            scale = torch.rand((cout,), device=dev, generator=g) + 0.5
            shift = torch.randn((cout,), device=dev, generator=g)
            kw.update(scale=scale, shift=shift)
        else:
            claims.append("AFFINE with scale = shift = NULL")
        kw["relu"] = True
        if "res" in o:
            roff, rwidth = o["res"]
            rbuf = _act(torch.randn((n, h, w, rwidth), device=dev, generator=g), split)
            res = rbuf[..., roff:roff + cout]
            kw["residual"] = res
            if rwidth != cout:
                claims.append("residual pitch %d != output pitch %d" % (rwidth, cout))
    out_f32 = None
    if epi == ops.EPI_F32:
        shift = torch.randn((cout,), device=dev, generator=g)
        kw["shift"] = shift
        if "oslice" in o:
            ooff, owidth = o["oslice"]
            obuf = torch.full((n, h, w, owidth), 7.0, device=dev)
            out_f32 = obuf[..., ooff:ooff + cout]
            kw["out_f32"] = out_f32
            claims.append("out_f32 = channels [%d, %d) of a %d-wide fp32 buffer (%s)" %
                          (ooff, ooff + cout, owidth, "8-byte aligned" if ooff % 2 == 0 else "odd float offset"))
    stats = bool(o.get("stats"))

    # geometry, tied to the library
    lib = _lib.load()
    k_slices = 1
    if split and epi != ops.EPI_F32:
        k_slices = int(lib.semseg_conv_k_slices(cin, len(taps), X3_MAX_KBLOCKS))
    geo = fprop_geom(n, h, w, cin, cout, len(taps), k_slices)
    assert geo["k_slices"] == k_slices
    assert ops.conv_stats_rows(n, h, w, cout) == 4 * min(geo["tiles"] * geo["n_tiles"], _sms())
    if split and epi != ops.EPI_F32:
        claims.append("%d K blocks -> %d slice(s) of <= %d" % (geo["kblocks"], k_slices, geo["kb_per_slice"]))
        if name.startswith("kslice"):
            want = {"8": 1, "9": 2, "18": 3, "576": 72}[name.split("-")[1]]
            assert geo["kblocks"] == int(name.split("-")[1]) and k_slices == want
    if geo["h"] % geo["bh"] or geo["w"] % geo["bw"]:
        claims.append("box %dx%d clips the %dx%d map" % (geo["bh"], geo["bw"], h, w))
    else:
        claims.append("box %dx%d tiles the %dx%d map exactly" % (geo["bh"], geo["bw"], h, w))
    if name.startswith("grid-61x67-clipped"):
        assert h % geo["bh"] and w % geo["bw"], "bottom- and right-clipped boxes"
        assert non_prefix_mask(geo), "W % bw != 0, so a statistics warp sees a non-prefix mask"
        if k_slices == 1:
            claims.append("W %% bw = %d: a statistics warp sees a non-prefix row mask" % (w % geo["bw"]))
    if name == "grid-3x5-below-one-box":
        assert geo["tiles"] == n and geo["bh"] * geo["bw"] == h * w < 128
    if name == "grid-n16-multi-item":
        assert k_slices == 1 and geo["items"] > _sms(), "items > SMs: a CTA accumulates several tiles into its rows"
        claims.append("%d items > %d SMs: CTAs accumulate several tiles" % (geo["items"], _sms()))
    if geo["n_tiles"] > 1 or cout % geo["block_n"]:
        claims.append("BLOCK_N %d, %d N tile(s), last one %d wide" %
                      (geo["block_n"], geo["n_tiles"], cout - (geo["n_tiles"] - 1) * geo["block_n"]))
    if name.startswith("cout320"):
        assert geo["n_tiles"] == 2 and cout % geo["block_n"]
    if name.startswith("cout192") or name.startswith("f32-15"):
        assert geo["block_n"] == 256 and geo["n_tiles"] == 1
    if epi == ops.EPI_F32:
        pitch = out_f32.stride(2) if out_f32 is not None else cout
        aligned = pitch % 2 == 0 and (out_f32 is None or out_f32.data_ptr() % 8 == 0)
        claims.append("out_pitch %d: %s stores" % (pitch, "float2" if aligned else "scalar"))
        if name.startswith("f32-19") or name.startswith("f32-21"):
            assert not aligned
    if cin % 64:
        claims.append("last K block holds %d of 64 channels" % (cin % 64))
    if dil >= h and dil >= w and k == 3:
        claims.append("dilation %d >= map %dx%d: every off-centre tap reads only halo" % (dil, h, w))

    def run():
        y, sp = ops.conv_fprop(x, slab, cout, taps, epi=epi, stats=stats, **kw)
        return (y.clone() if out_f32 is None else obuf.clone()), (sp.clone() if sp is not None else None)

    y1, sp1 = run()
    y2, sp2 = run()
    assert torch.equal(y1, y2) and (sp1 is None or torch.equal(sp1, sp2)), "not bit-identical on a second call"
    if out_f32 is not None:
        outside = torch.ones(owidth, dtype=torch.bool, device=dev)
        outside[ooff:ooff + cout] = False
        assert bool((y1[..., outside] == 7.0).all()), "F32 epilogue wrote outside its channel slice"
        y1 = y1[..., ooff:ooff + cout]

    # reference
    xp, wp = planes(x, split), planes(slab, split)
    ref, s = seg_conv(xp, wp, taps, cout)
    steps = C_TRUNC * geo["kb_per_slice"] * 4 * nseg + (k_slices if k_slices > 1 else 0)
    if epi == ops.EPI_F32:
        r_out = R_F32
    else:
        r_out = R_SPLIT if split else R_BF16

    def finish(ref, s, with_res=True):
        """(value, S, extra fp32 roundings) after the epilogue."""
        if epi == ops.EPI_F32:
            return ref + shift.double(), s + shift.double().abs(), 1
        if epi == ops.EPI_AFFINE:
            if scale is not None:
                ref, s = ref * scale.double(), s * scale.double().abs()
            if shift is not None:
                ref, s = ref + shift.double(), s + shift.double().abs()
            if res is not None and with_res:
                ref, s = ref + stored(res), s + stored(res).abs()
            return ref.clamp_min(0.0), s, 3
        return ref, s, 0

    fref, fs, extra = finish(ref, s)
    out = stored(y1)
    worst = ratio(out, fref, fs, r_out, steps + extra)

    # teeth: the reference without the guarded contribution
    t = o["teeth"]
    tref, ts = ref, s
    if t == "tap":
        tref, ts = seg_conv(xp, wp, taps[:-1], cout)
        claims.append("teeth: tap %s dropped" % (taps[-1],))
    elif t == "halo":   # an off-centre tap that read the pixel under the centre instead of the halo zeros
        xr, sr = seg_conv(xp, wp, [(0, 0, taps[0][2])], cout)
        tref, ts = ref + xr, s + sr
        claims.append("teeth: tap %s reads the centre pixel instead of halo" % (taps[0],))
    elif t == "kblock":
        kb0 = 64 * ((cin - 1) // 64)
        xcut = [p.clone() for p in xp]
        for p in xcut:
            p[..., kb0:] = 0
        tref, ts = seg_conv(xcut, wp, taps, cout)
        claims.append("teeth: K block of channels [%d, %d) dropped" % (kb0, cin))
    elif t in ("box", "ntile", "lastch"):
        tref, ts = ref.clone(), s.clone()
        if t == "box":            # the last pixel box of the last image was never stored
            bh, bw = geo["bh"], geo["bw"]
            hh0, ww0 = (cdiv(h, bh) - 1) * bh, (cdiv(w, bw) - 1) * bw
            tref[-1, hh0:, ww0:] = 0
            ts[-1, hh0:, ww0:] = 0
            claims.append("teeth: last box (rows %d.., cols %d..) not stored" % (hh0, ww0))
        else:
            c0 = (geo["n_tiles"] - 1) * geo["block_n"] if t == "ntile" else cout - 1
            if t == "ntile" and geo["n_tiles"] == 1:
                c0 = 64 * ((cout - 1) // 64)        # the last (partial) 64-column chunk of the only N tile
            tref[..., c0:] = 0
            ts[..., c0:] = 0
            claims.append("teeth: output channels [%d, %d) not stored" % (c0, cout))
    else:
        assert t == "res"
        claims.append("teeth: residual not added")
    teeth_ref, teeth_s, _ = finish(tref, ts, with_res=t != "res")
    teeth = ratio(out, teeth_ref, teeth_s, r_out, steps + extra)

    if stats:
        m = n * h * w
        if k_slices > 1:
            rows = splitk_chunk_rows(m)
            assert int(lib.semseg_conv_splitk_rows(m)) == cdiv(m, rows) == sp1.shape[0]
            depth = rows // 32 + 32 + 1
            claims.append("statistics from the K-slice finish: %d chunk rows" % sp1.shape[0])
        else:
            assert sp1.shape[0] == 4 * geo["grid"]
            depth = 32 + cdiv(geo["items"], geo["grid"]) + 1
        cnt = sp1.double()[:, 2].sum(0)
        assert bool((cnt == m).all()), "statistics count %s != N*H*W = %d" % (cnt.unique().tolist(), m)
        y64 = out.reshape(m, cout)
        sworst = _stats_ratio(sp1, y64, depth)
        steeth = _stats_ratio(sp1, y64[:-1], depth)   # the last pixel of the map left out of the statistics
        claims.append("statistics worst %.3g, teeth %.3g" % (sworst, steeth))
        assert sworst <= 1.0 and steeth > 1.0
    report(name + ("-x3" if split else "-bf16"), claims, worst, teeth)


# ------------------------------------------------------------------------------------------------ stride 2 (phases)
@pytest.mark.parametrize("split", [False, True], ids=["bf16", "x3"])
@pytest.mark.parametrize("n,h,w,cin,cout,k", [(2, 13, 13, 64, 64, 3), (1, 12, 10, 64, 128, 3), (2, 11, 8, 128, 64, 1),
                                              (1, 9, 14, 24, 64, 3)])
def test_conv_stride2_phases_vs_float64_conv(n, h, w, cin, cout, k, split):
    """fprop and wgrad of a stride-2 conv through space_to_phases + conv_taps_s2 (img_add), element by element against
    float64 F.conv2d(stride=2) and its weight gradient, on the operands the kernels read."""
    from semseg_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(n * 1000 + h * 10 + w)
    nseg = 3 if split else 1
    x = _act(torch.randn((n, h, w, cin), device="cuda", generator=g), split)
    wt = torch.randn((cout, cin, k, k), device="cuda", generator=g) / (cin * k * k) ** 0.5
    pw = ops.pack_weights(wt, split=split)
    xp = ops.space_to_phases(x)
    t2 = ops.conv_taps_s2(k, n)
    taps, img_add = [t[:3] for t in t2], [t[3] for t in t2]
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    y1, _ = ops.conv_fprop(xp, pw.wf, cout, taps, img_add=img_add, out_nhw=(n, ho, wo))
    y2, _ = ops.conv_fprop(xp, pw.wf, cout, taps, img_add=img_add, out_nhw=(n, ho, wo))
    assert torch.equal(y1, y2)

    def nchw(t):
        return t.permute(0, 3, 1, 2)

    def oihw(slab):   # wf[r*k + s][co][ci] -> [co][ci][r][s]
        return slab[:, :, :cin].reshape(k, k, cout, cin).permute(2, 3, 0, 1)

    xs, ws = planes(x, split), planes(pw.wf, split)
    ref = s = 0
    for xa, wa in _segments(xs, ws):
        ref = ref + F.conv2d(nchw(xa), oihw(wa), stride=2, padding=k // 2)
        s = s + F.conv2d(nchw(xa).abs(), oihw(wa).abs(), stride=2, padding=k // 2)
    ref, s = ref.permute(0, 2, 3, 1), s.permute(0, 2, 3, 1)
    kb = len(taps) * cdiv(cin, 64)
    k_slices = cdiv(kb, cdiv(kb, cdiv(kb, X3_MAX_KBLOCKS))) if split else 1
    steps = C_TRUNC * cdiv(kb, k_slices) * 4 * nseg + (k_slices if k_slices > 1 else 0)
    r_out = R_SPLIT if split else R_BF16
    out = stored(y1)
    worst = ratio(out, ref, s, r_out, steps)
    # the tap mirror on the phase tensor is the same convolution
    pref, _ = seg_conv(planes(xp, split), ws, taps, cout, img_add, (n, ho, wo))
    assert float((pref - ref).abs().max()) <= 1e-9 * float(s.max())
    # teeth: every tap reads the next phase image (img_add off by N)
    tref, ts = seg_conv(planes(xp, split), ws, taps, cout, [(a + n) % (4 * n) for a in img_add], (n, ho, wo))
    teeth = ratio(out, tref, ts, r_out, steps)

    # wgrad on the phase tensor (img_add), the library's split choice
    dy = _act(torch.randn((n, ho, wo, cout), device="cuda", generator=g), split)
    dw1 = ops.conv_wgrad(xp, dy, cin, cout, taps, img_add=img_add)
    dw2 = ops.conv_wgrad(xp, dy, cin, cout, taps, img_add=img_add)
    assert torch.equal(dw1, dw2)
    geo = wgrad_geom(n, ho, wo, cin, cout, len(taps), split)

    def wgrad_ref(dy_planes):
        wref = ws_ = 0
        for dya, xa in _segments(dy_planes, xs):
            wref = wref + torch.nn.grad.conv2d_weight(nchw(xa), (cout, cin, k, k), nchw(dya), stride=2, padding=k // 2)
            ws_ = ws_ + torch.nn.grad.conv2d_weight(nchw(xa).abs(), (cout, cin, k, k), nchw(dya).abs(), stride=2,
                                                    padding=k // 2)
        return wref, ws_

    wsteps = C_TRUNC * geo["boxes_per_split"] * 4 * nseg + geo["n_splits"]
    wworst = ratio(dw1.double(), *wgrad_ref(planes(dy, split)), R_F32, wsteps)
    cut = [p.clone() for p in planes(dy, split)]
    for p in cut:            # teeth: the last output row of the last image left out of the pixel sum
        p[-1, -1] = 0
    wteeth = ratio(dw1.double(), *wgrad_ref(cut), R_F32, wsteps)
    report("stride2-%dx%d-k%d-%s" % (h, w, k, "x3" if split else "bf16"),
           ["%s sizes, output %dx%d" % ("odd" if h % 2 else "even", ho, wo),
            "wgrad: %d splits of <= %d boxes, worst %.3g" % (geo["n_splits"], geo["boxes_per_split"], wworst)],
           max(worst, wworst), min(teeth, wteeth))


# ------------------------------------------------------------------------------------------------ wgrad
def wgrad_run(x, dy, cin, cout, taps, n_splits):
    """semseg_conv_wgrad with an explicit split count (0 = the library's choice) and partials pre-filled with NaN (every
    element must be written), reduced by semseg_wgrad_reduce. Returns (dW OIHW, n_splits)."""
    from semseg_b200 import ops, _lib
    lib = _lib.load()
    nin, hin, win, _, xp = ops._nhwc_meta(x)
    n, h, w, _, dp = ops._nhwc_meta(dy)
    d = _lib.WgradDesc()
    d.N, d.H, d.W, d.Cin, d.Cout = n, h, w, cin, cout
    d.x, d.Nin, d.Hin, d.Win, d.x_pitch = x.data_ptr(), nin, hin, win, xp
    d.dy, d.dy_pitch = dy.data_ptr(), dp
    d.x_lo, d.dy_lo = ops._lo_int(x), ops._lo_int(dy)
    ops._fill_taps(d, taps, with_wtap=False)
    d.n_splits = n_splits
    splits = int(lib.semseg_conv_wgrad_splits(ctypes.byref(d)))
    assert splits > 0
    part = torch.full((splits, len(taps), cout, cin), float("nan"), device=x.device)
    d.dw_partial, d.n_splits = part.data_ptr(), splits
    _lib.check(lib.semseg_conv_wgrad(ctypes.byref(d), ops._stream()), "semseg_conv_wgrad")
    assert not bool(part.isnan().any()), "wgrad left partial elements unwritten"
    k = int(round(len(taps) ** 0.5))
    dw = torch.empty((cout, cin, k, k), device=x.device)
    _lib.check(lib.semseg_wgrad_reduce(ops._ptr(part), splits, len(taps), cout, cin, ops._ptr(dw), 0, ops._stream()),
               "semseg_wgrad_reduce")
    return dw, splits


def wgrad_ref(x_planes, dy_planes, taps, cout):
    """(dW, S) OIHW float64: dW[co][ci][t] = sum_p dy[p, co] * x[p + off(t), ci] over the kernel's segments."""
    cin = x_planes[0].shape[-1]
    out = []
    for absval in (False, True):
        acc = 0
        for dya, xa in _segments(dy_planes, x_planes):
            if absval:
                dya, xa = dya.abs(), xa.abs()
            m = dya.reshape(-1, dya.shape[-1])[:, :cout]
            acc = acc + torch.stack([m.t() @ _shift(xa, dh, dw, 0, tuple(dya.shape[:3])).reshape(-1, cin)
                                     for dh, dw, _ in taps], -1)
        k = int(round(len(taps) ** 0.5))
        out.append(acc.reshape(cout, cin, k, k))
    return out


# id: (N, H, W, Cin, Cout, k, dilation, teeth)
WGRAD = {
    "cls-cout24": (2, 9, 11, 512, 24, 1, 1, "lastco"),
    "cls-cout152-second-co-tile": (2, 9, 11, 512, 152, 1, 1, "cotile"),
    "cin64-units-4-4-1": (2, 13, 11, 64, 64, 3, 1, "lasttap"),
    "cin128-units-2-2-2-2-1": (2, 13, 11, 128, 64, 3, 2, "lasttap"),
    "cin32-3x3": (2, 9, 9, 32, 64, 3, 1, "lasttap"),
    "cin192-cout192": (1, 9, 10, 192, 192, 3, 1, "lastci"),
    "cin256-cout320": (1, 8, 9, 256, 320, 1, 1, "cotile"),
    "cin512-3x3-d4": (1, 9, 9, 512, 64, 3, 4, "lasttap"),
    "cin4096-3x3": (1, 6, 7, 4096, 64, 3, 1, "lasttap"),
    "x3-21-box-bound": (1, 40, 40, 256, 128, 1, 1, "box"),
    "grid-61x67": (1, 61, 67, 64, 64, 3, 1, "box"),
    "grid-h1-w300": (1, 1, 300, 64, 64, 1, 1, "box"),
    "grid-h300-w1": (1, 300, 1, 128, 64, 1, 1, "box"),
    "grid-3x5": (2, 3, 5, 64, 128, 3, 1, "lasttap"),
    "grid-n16": (16, 12, 12, 64, 64, 3, 1, "box"),
}


@pytest.mark.parametrize("split", [False, True], ids=["bf16", "x3"])
@pytest.mark.parametrize("name", list(WGRAD))
def test_conv_wgrad_element_bound(name, split):
    """wgrad + wgrad_reduce against float64 at the library's split count, one split and one pixel box per split."""
    from semseg_b200 import ops
    n, h, w, cin, cout, k, dil, t = WGRAD[name]
    g = torch.Generator(device="cuda").manual_seed(hash(name) % 10007)
    nseg = 3 if split else 1
    x = _act(torch.randn((n, h, w, cin), device="cuda", generator=g), split)
    dy = _act(torch.randn((n, h, w, cout), device="cuda", generator=g), split)
    taps = ops.conv_taps(k, dil)
    geo = wgrad_geom(n, h, w, cin, cout, len(taps), split)
    claims = ["%d boxes, %d co tile(s), BLOCK_N %d, %d ci tile(s)" %
              (geo["boxes"], geo["co_tiles"], geo["block_n"], geo["ci_tiles"])]
    if geo["tu"] > 1:
        claims.append("tap units %s" % geo["unit_sizes"])
    if name == "cin64-units-4-4-1":
        assert geo["unit_sizes"] == [4, 4, 1], "Cin = 64: units of 4, 4 and 1 taps"
    if name == "cin128-units-2-2-2-2-1":
        assert geo["unit_sizes"] == [2, 2, 2, 2, 1], "Cin = 128: five units, the last with a single tap"
    if t == "cotile":
        assert geo["co_tiles"] >= 2 and cout % 128, "a partial second (or later) co tile"
    if t == "lastci":
        assert cin % geo["block_n"], "a partial last ci tile"
    if name == "x3-21-box-bound" and split:
        free = wgrad_geom(n, h, w, cin, cout, len(taps), False)
        assert geo["n_splits"] > free["n_splits"], "the 21-box bound raises the split count"
        claims.append("21-box bound: %d splits instead of %d" % (geo["n_splits"], free["n_splits"]))
    xs, dys = planes(x, split), planes(dy, split)
    ref, s = wgrad_ref(xs, dys, taps, cout)
    if t == "lasttap":
        tref, ts = ref.clone(), s.clone()
        tref.view(cout, cin, -1)[..., -1] = 0
        ts.view(cout, cin, -1)[..., -1] = 0
    elif t in ("cotile", "lastco"):
        c0 = 128 * (geo["co_tiles"] - 1) if t == "cotile" else cout - 1
        tref, ts = ref.clone(), s.clone()
        tref[c0:] = 0
        ts[c0:] = 0
    elif t == "lastci":
        c0 = geo["block_n"] * (geo["ci_tiles"] - 1) + 64 * ((cin % geo["block_n"] - 1) // 64)
        tref, ts = ref.clone(), s.clone()
        tref[:, c0:] = 0
        ts[:, c0:] = 0
    else:
        assert t == "box"
        bh, bw = choose_box(h, w, 64)
        cut = [p.clone() for p in dys]
        for p in cut:
            p[-1, (cdiv(h, bh) - 1) * bh:, (cdiv(w, bw) - 1) * bw:] = 0
        tref, ts = wgrad_ref(xs, cut, taps, cout)
    worst, teeth = 0.0, math.inf
    for label, want in (("library", 0), ("one split", 1), ("one box per split", geo["boxes"])):
        gs = wgrad_geom(n, h, w, cin, cout, len(taps), split, want)
        dw1, splits = wgrad_run(x, dy, cin, cout, taps, want)
        dw2, _ = wgrad_run(x, dy, cin, cout, taps, want)
        assert torch.equal(dw1, dw2), "not bit-identical on a second call"
        assert splits == gs["n_splits"], "split mirror disagrees with semseg_conv_wgrad_splits"
        if want == 0:
            assert torch.equal(dw1, ops.conv_wgrad(x, dy, cin, cout, taps))
            if split:
                assert gs["boxes_per_split"] <= 21, "bf16x3 chains are bounded to 21 pixel boxes"
        steps = C_TRUNC * gs["boxes_per_split"] * 4 * nseg + splits
        r = ratio(dw1.double(), ref, s, R_F32, steps)
        worst = max(worst, r)
        teeth = min(teeth, ratio(dw1.double(), tref, ts, R_F32, steps))
        claims.append("%s: %d split(s) x <= %d boxes, worst %.3g" % (label, splits, gs["boxes_per_split"], r))
    claims.append("teeth: %s" % t)
    report("wgrad-%s-%s" % (name, "x3" if split else "bf16"), claims, worst, teeth)


@pytest.mark.parametrize("n_splits,taps,cout,cin,accumulate", [
    (1, 1, 64, 64, 0), (5, 9, 24, 512, 1), (9, 9, 152, 64, 0), (70, 9, 64, 64, 1),
    (3, 9, 3, 5, 0), (7, 1, 19, 9, 1), (4, 4, 7, 13, 0)])
def test_wgrad_reduce_vs_float64(n_splits, taps, cout, cin, accumulate):
    """semseg_wgrad_reduce on random partials: the vector variant (Cout*Cin % 4 == 0), the scalar one (reachable only
    through the ABI) and accumulate=1, against a float64 sum; nothing past the output is written."""
    from semseg_b200 import ops, _lib
    lib = _lib.load()
    g = torch.Generator(device="cuda").manual_seed(n_splits * 100 + cin)
    part = torch.randn((n_splits, taps, cout, cin), device="cuda", generator=g)
    plane = cout * cin
    old = torch.randn((plane * taps,), device="cuda", generator=g)
    buf = torch.full((plane * taps + 64,), 7.0, device="cuda")

    def run():
        buf[:plane * taps] = old
        _lib.check(lib.semseg_wgrad_reduce(ops._ptr(part), n_splits, taps, cout, cin, ops._ptr(buf), accumulate,
                                           ops._stream()), "semseg_wgrad_reduce")
        return buf.clone()

    out1, out2 = run(), run()
    assert torch.equal(out1, out2)
    assert bool((out1[plane * taps:] == 7.0).all()), "wrote past the output"
    p64 = part.double().permute(2, 3, 1, 0)             # [co][ci][t][split]
    ref = p64.sum(-1).reshape(-1) + (old.double() if accumulate else 0)
    s = p64.abs().sum(-1).reshape(-1) + (old.double().abs() if accumulate else 0)
    steps = n_splits + accumulate
    worst = ratio(out1[:plane * taps].double(), ref, s, 0.0, steps)
    tref = p64[..., :-1].sum(-1).reshape(-1) + (old.double() if accumulate else 0)   # the last split dropped
    teeth = ratio(out1[:plane * taps].double(), tref, s, 0.0, steps)
    report("wgrad_reduce-%dx%dx%dx%d" % (n_splits, taps, cout, cin),
           ["%s variant" % ("vector" if plane % 4 == 0 else "scalar"), "accumulate=%d" % accumulate],
           worst, teeth)


# ------------------------------------------------------------------------------------------------ classifier
@pytest.mark.parametrize("split", [False, True], ids=["bf16", "x3"])
@pytest.mark.parametrize("classes", [19, 21, 150])
def test_classifier_conv_bias_f32_forward_backward(classes, split):
    """functional.conv_bias_f32 (the cls / aux 1x1 classifier) forward and backward (dx, dW, db) element by element
    against float64 on the exact operands: x as stored, the cached wf / wd slabs, dy as converted for the backward."""
    from semseg_b200 import functional, ops
    n, h, w, cin = 2, 9, 11, 512
    g = torch.Generator(device="cuda").manual_seed(classes)
    nseg = 3 if split else 1
    torch.manual_seed(classes)
    conv = torch.nn.Conv2d(cin, classes, 1).cuda()
    x = _act(torch.randn((n, h, w, cin), device="cuda", generator=g), split).requires_grad_(True)
    y = functional.conv_bias_f32(x, conv)
    dy = torch.randn(y.shape, device="cuda", generator=g)
    y.backward(dy)
    pw = functional.packed(conv, split=split)
    cp = pw.wd.shape[-1]
    assert cp == ops.round_up(classes, 8)
    dyb = ops.f32_to_act(dy, split)            # the operand the backward's dgrad and wgrad read
    xs = planes(x.detach(), split)
    m = n * h * w
    claims = ["dgrad Cin = %d (last K block %d of 64 channels)" % (cp, cp % 64)]

    # forward: F32 epilogue, out_pitch = classes (odd for 19 / 21: scalar stores)
    ref, s = seg_conv(xs, planes(pw.wf, split), ops.conv_taps(1, 1), classes)
    b = conv.bias.detach().double()
    steps = C_TRUNC * cdiv(cin, 64) * 4 * nseg + 1
    yw = ratio(y.detach().double(), ref + b, s + b.abs(), R_F32, steps)
    yt = ratio(y.detach().double(), torch.cat([ref[..., :-1], 0 * ref[..., -1:]], -1) + b, s + b.abs(), R_F32, steps)
    claims.append("forward out_pitch %d (%s stores)" % (classes, "scalar" if classes % 2 else "float2"))

    # dx: dgrad of the padded dy on the wd slab, bf16 / hi-lo output
    dref, ds = seg_conv(planes(dyb, split), planes(pw.wd, split), ops.conv_taps(1, 1), cin)
    dsteps = C_TRUNC * cdiv(cp, 64) * 4 * nseg
    r_act = R_SPLIT if split else R_BF16
    xg = stored(x.grad)
    dxw = ratio(xg, dref, ds, r_act, dsteps)
    cut = [p.clone() for p in planes(dyb, split)]
    for p in cut:
        p[..., 64 * ((cp - 1) // 64):] = 0     # the last (partial) K block dropped
    dxt = ratio(xg, *seg_conv(cut, planes(pw.wd, split), ops.conv_taps(1, 1), cin), r_act, dsteps)

    # dW: wgrad with Cout = cp, rows >= classes dropped by the module
    wr, wsum = wgrad_ref(xs, planes(dyb, split), ops.conv_taps(1, 1), cp)
    geo = wgrad_geom(n, h, w, cin, cp, 1, split)
    wsteps = C_TRUNC * geo["boxes_per_split"] * 4 * nseg + geo["n_splits"]
    gw = conv.weight.grad.double()
    dww = ratio(gw, wr[:classes], wsum[:classes], R_F32, wsteps)
    c0 = 128 if classes > 128 else classes - 1   # the second, partial co tile (150) or the last class
    dwt = ratio(gw, torch.cat([wr[:c0], 0 * wr[c0:classes]]), torch.cat([wsum[:c0], 0 * wsum[c0:classes]]), R_F32,
                wsteps)
    claims.append("wgrad Cout = %d: %d co tile(s), %d split(s)" % (cp, geo["co_tiles"], geo["n_splits"]))
    if classes == 150:
        assert geo["co_tiles"] == 2 and cp % 128

    # db: fp32 sum over the pixels
    dbw = ratio(conv.bias.grad.double(), dy.double().sum((0, 1, 2)), dy.double().abs().sum((0, 1, 2)), 0.0, m)
    dbt = ratio(conv.bias.grad.double(), dy.double()[:, :, :-1].sum((0, 1, 2)), dy.double().abs().sum((0, 1, 2)), 0.0,
                m)
    claims.append("worst y %.3g dx %.3g dW %.3g db %.3g" % (yw, dxw, dww, dbw))

    # a second forward / backward gives the same bits
    x2 = x.detach().clone().requires_grad_(True)
    conv.weight.grad = conv.bias.grad = None
    y2 = functional.conv_bias_f32(x2, conv)
    y2.backward(dy)
    assert torch.equal(y2, y) and torch.equal(x2.grad, x.grad)
    assert torch.equal(conv.weight.grad.double(), gw)
    report("classifier-%d-%s" % (classes, "x3" if split else "bf16"), claims, max(yw, dxw, dww, dbw),
           min(yt, dxt, dwt, dbt))


# ------------------------------------------------------------------------------------------------ rejected geometry
def test_misaligned_residual_rejected_before_launch():
    """The epilogues read the residual as bf16 pairs (fprop) or 16-byte vectors (K-slice finish): a residual slice that
    breaks that alignment is SEMSEG_E_INVALID, not a misaligned access."""
    from semseg_b200 import ops, _lib
    g = torch.Generator(device="cuda").manual_seed(5)
    for split, off in ((False, 1), (True, 4)):
        x = _act(torch.randn((1, 5, 6, 64), device="cuda", generator=g), split)
        pw = ops.pack_weights(torch.randn((64, 64, 3, 3), device="cuda", generator=g) * 0.05, split=split)
        rbuf = _act(torch.randn((1, 5, 6, 136), device="cuda", generator=g), split)
        res = rbuf[..., off:off + 64]
        with pytest.raises(_lib.SemsegError, match="aligned"):
            ops.conv_fprop(x, pw.wf, 64, ops.conv_taps(3, 1), epi=ops.EPI_AFFINE, residual=res)
        torch.cuda.synchronize()
