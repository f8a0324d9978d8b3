"""GPU tier (-m gpu): the batch-statistics BatchNorm kernels of csrc/bn.cu (statistics merge and finalise, the NCCL-form
finalise, apply, the two backward passes) and the split-aware element-wise ops (add_act, scale_nc, f32_to_act,
act_to_f32) element by element at their chunk, channel-group and pitch edges. Conventions as in test_conv_edges_gpu.py,
whose helpers are used here.

Reference. float64 on exactly what the kernel reads: the stored activation values (bf16, or the fp32 sum hi + lo that
act_unpack forms), the fp32 statistics table, and for a kernel that consumes an earlier kernel's coefficients, those
coefficients (apply gets the finalise's scale_shift, bwd_apply the kernel's sums and mean_invstd), so every kernel is
held to its own operation order. u = 2^-24.

Bounds (each derived next to the kernel lines it covers, see the functions below):
  finalise   the block merge adds raw (S, Q, n) over a thread's rows and the lanes of its warp, forms mean = S/n and
             M2 = Q - S*mean once per warp, then merges the 32 warps with Chan's formula in a 5-level tree. The
             error is propagated through exactly that order (`_merge_bound`), so the variance bound carries the
             depth*u*sum(y^2) term of the raw-moment form, not only depth*u*M2;
  apply      fmaf(x, sc, sh) + r: 2u*(|x*sc| + |sh| + |r|);
  bwd_reduce (rows_per_chunk/32 + 32 + chunks + 3)*u*sum|term|;
  bwd_apply  10u*(|ka*dz| + |kx*x| + |ka*s1/M| + |kx*mean|): the roundings of ka, kx, kb and the two fmas;
  outputs    bf16: the stored value is the round-to-nearest of some value within the bound; split: + 2^-16*|ref|.
The ReLU mask is exact: the value the kernel reads has at most 24 significant bits, so x*sc is exact in float64 and
adding the fp32 shift cannot change its sign; the float64 sign of x*sc + sh is the sign of the kernel's fmaf.

Teeth. Each case recomputes the reference without the contribution it guards (the last table row, the last backward
chunk, the last pixel, the last 8-channel group or partial 64-channel block, the residual, the ReLU mask) and asserts
that the same bound flags at least one element.

Geometry. chunk_rows, stats_group_channels and ew_grid / ew_grid_fixed_channels are mirrored here and tied to the
library through semseg_bn_workspace_floats; each case asserts the branch it names.
"""
import numpy as np
import pytest
import torch

from tests.test_conv_edges_gpu import R_BF16, R_SPLIT, U, _act, _sms, cdiv, ratio, report, stored

pytestmark = pytest.mark.gpu

EPS = float(np.float32(1e-5))        # what the kernels receive as `float eps` / `float momentum`
MOM = float(np.float32(0.1))
SENTINEL = 7.0


@pytest.fixture(scope="module", autouse=True)
def _device():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    yield


# ------------------------------------------------------------------------------------------------ geometry mirror
def chunk_rows(m):
    """csrc/bn.cu::chunk_rows: pixel rows per backward chunk."""
    return (max(cdiv(m, 1024), 256) + 31) & ~31


def stats_group_channels(c):
    """csrc/bn.cu::stats_group_channels: channels per 1024-thread statistics block (the CH template argument)."""
    return 8 if c <= 1024 else (16 if c <= 2048 else 32)


def ew_grid(total, threads=256):
    """csrc/bn.cu::ew_grid."""
    return max(min(cdiv(total, threads), _sms() * 16), 1)


def ew_grid_fixed_channels(total, threads, groups):
    """csrc/bn.cu::ew_grid_fixed_channels: grid * threads is a multiple of groups = C/8."""
    m = 1
    while (m * threads) % groups:
        m += 1
    return cdiv(ew_grid(total, threads), m) * m


def stride_passes(m, c, unroll):
    """(pixel stride, most passes of a thread, whether some thread runs the non-unrolled tail) of the fixed-channel
    grid-stride loops of bn_apply (unroll 4) and bn_bwd_apply (unroll 2)."""
    groups = c // 8
    pstride = ew_grid_fixed_channels(m * groups, 256, groups) * 256 // groups
    counts = [cdiv(m - p0, pstride) for p0 in range(min(pstride, m))]
    return pstride, max(counts), any(k % unroll for k in counts)


def _lib():
    from semseg_b200 import _lib as L
    return L.load()


def test_geometry_mirror_tied_to_library():
    lib = _lib()
    for m in (1, 2, 31, 256, 257, 7200, 80000, 262144, 1 << 20):
        for c in (8, 72, 2048):
            assert lib.semseg_bn_workspace_floats(m, c) == cdiv(m, chunk_rows(m)) * 2 * c, (m, c)
    assert cdiv(80000, chunk_rows(80000)) == 313


# ------------------------------------------------------------------------------------------------ helpers
def worst_ratio(out, ref, bound):
    """max |out - ref| / bound over the elements (fp32 outputs: no storage term); a zero bound admits only 0."""
    out, ref, bound = out.double(), ref.double(), bound.double()
    err = (out - ref).abs()
    r = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, torch.inf, 0.0))
    return float(r.max())


def act_ratio(out, ref, s, steps, split):
    return ratio(stored(out), ref, s, R_SPLIT if split else R_BF16, steps)


def pixels(t):
    """[M, C] float64 view of an activation's stored values (M = N*H*W)."""
    v = stored(t)
    return v.reshape(-1, v.shape[-1])


def in_buffer(m, c, split, gen, off=None, width=None, scale=1.0, shift=0.0):
    """An activation [1, 1, M, C] (pitch C), or channels [off, off + C) of a [1, 1, M, width] buffer; the rest of the
    buffer holds other values."""
    w = c if off is None else width
    buf = _act(torch.randn((1, 1, m, w), device="cuda", generator=gen) * scale + shift, split)
    return (buf, buf if off is None else buf[..., off:off + c])


def out_buffer(m, c, split, off=None, width=None):
    """(buffer, view): the view is what the kernel writes; the buffer is filled with a sentinel."""
    from semseg_b200 import ops
    w = c if off is None else width
    buf = ops.empty_act((1, 1, m, w), split, "cuda").fill_(SENTINEL)
    return buf, (buf if off is None else buf[..., off:off + c])


def assert_outside_untouched(buf, off, c):
    if off is None:
        return
    keep = torch.ones(buf.shape[-1], dtype=torch.bool, device=buf.device)
    keep[off:off + c] = False
    assert bool((buf[..., keep].float() == SENTINEL).all()), "a kernel wrote outside its channel slice"


def coefficients(x, gen, gamma=True):
    """(mean_invstd [3][C], scale_shift [2][C], gamma, beta) of x from the finalise kernel, fed a one-row table of x's
    moments."""
    from semseg_b200 import ops
    v = pixels(x)
    c = v.shape[1]
    table = torch.stack([v.sum(0), (v * v).sum(0), torch.full((c,), float(v.shape[0]), device="cuda",
                                                              dtype=torch.float64)]).float()[None]
    g = torch.rand((c,), device="cuda", generator=gen) + 0.5 if gamma else None
    b = torch.randn((c,), device="cuda", generator=gen)
    mi, ss = ops.bn_finalize_partials(table, g, b, EPS, MOM, None, None)
    return mi, ss, g, b


# ------------------------------------------------------------------------------------------------ finalise
def synthetic_table(t, c, gen, ratios=(0.0, 1.0, 30.0)):
    """[T][3][C] fp32 (sum, sum of squares, count) rows of virtual data with mean/std ratio cycling over `ratios` by
    channel: counts 1..64 with every 8th row (never the last) empty, row means and M2 drawn as a sample of that size
    would give them."""
    sig = torch.exp(0.5 * torch.randn((c,), device="cuda", generator=gen, dtype=torch.float64))
    mu = sig * torch.tensor(ratios, device="cuda", dtype=torch.float64).repeat(cdiv(c, len(ratios)))[:c]
    n = torch.randint(1, 65, (t, 1), device="cuda", generator=gen).double().expand(t, c).clone()
    n[torch.arange(t, device="cuda") % 8 == 3] = 0
    n[-1] = n[-1].clamp_min(1)
    z = torch.randn((t, c), device="cuda", generator=gen, dtype=torch.float64)
    mean_t = mu + sig * z / n.clamp_min(1).sqrt()
    m2_t = sig ** 2 * (n - 1).clamp_min(0) * (1 + 0.3 * torch.randn((t, c), device="cuda", generator=gen,
                                                                       dtype=torch.float64)).abs()
    s = n * mean_t
    q = m2_t + n * mean_t ** 2
    return torch.stack([s, q, n], 1).float().contiguous(), torch.tensor(ratios * cdiv(c, len(ratios)))[:c]


def _warp_moments(tab, ch):
    """block_conv_moments up to the per-warp (n, mean, M2), in float64, with first-order error bounds (em, e2) of the
    kernel's fp32 values. Row t goes to thread row lane t % RL (RL = 1024/CH), i.e. to warp (t % RL) // (32/CH).

        S += row[c]; Q += row[C + c]; n += row[2C + c]     R = ceil(T/RL) rows per lane, then log2(32/CH) butterfly
            -> |dS| <= (R + 32/CH) u sum|S_t|, |dQ| <= (R + 32/CH) u sum Q_t   (every partial sum is below the sum of
               absolute values; n is exact: integers < 2^24)
        mean = S / n                                      -> em = |dS|/n + u|mean|
        m2 = fmaxf(Q - S * mean, 0)                       -> e2 = |dQ| + |S| em + |mean| |dS| + u|S mean| + u|m2|
    """
    t, _, c = tab.shape
    rl = 1024 // ch
    depth = cdiv(t, rl) + 32 // ch
    tb = tab.double()
    warp = (torch.arange(t, device="cuda") % rl) // (32 // ch)
    def per_warp(v):
        return torch.zeros((32, c), device="cuda", dtype=torch.float64).index_add_(0, warp, v)
    s, q, n = per_warp(tb[:, 0]), per_warp(tb[:, 1]), per_warp(tb[:, 2])
    ds = depth * U * per_warp(tb[:, 0].abs())
    dq = depth * U * q
    nz = n > 0
    mean = torch.where(nz, s / n.clamp_min(1), 0.0)
    m2 = torch.where(nz, (q - s * mean).clamp_min(0), 0.0)
    em = torch.where(nz, ds / n.clamp_min(1) + U * mean.abs(), 0.0)
    e2 = torch.where(nz, dq + s.abs() * em + mean.abs() * ds + U * (s * mean).abs() + U * m2, 0.0)
    return dict(n=n, mean=mean, m2=m2, em=em, e2=e2), depth


def _merge_bound(a, b):
    """merge() of csrc/bn.cu in float64 with propagated bounds:
        d = b.mean - a.mean                               -> ed = em_a + em_b + u|d|
        mean = a.mean + d * (b.n / n)                     -> em = em_a + f ed + 3u(|d f| + |mean|),  f = b.n / n
        m2 = a.m2 + b.m2 + d * d * (a.n * b.n / n)        -> e2 = e2_a + e2_b + w(2|d| ed + ed^2) + 5u w d^2 + 2u m2
    and the two early returns for an empty side."""
    n = a["n"] + b["n"]
    f = torch.where(n > 0, b["n"] / n.clamp_min(1), 0.0)
    w = torch.where(n > 0, a["n"] * b["n"] / n.clamp_min(1), 0.0)
    d = b["mean"] - a["mean"]
    ed = a["em"] + b["em"] + U * d.abs()
    mean = a["mean"] + d * f
    m2 = a["m2"] + b["m2"] + d * d * w
    r = dict(n=n, mean=mean, m2=m2, em=a["em"] + f * ed + 3 * U * ((d * f).abs() + mean.abs()),
             e2=a["e2"] + b["e2"] + w * (2 * d.abs() * ed + ed * ed) + 5 * U * w * d * d + 2 * U * m2)
    for k in r:
        r[k] = torch.where(b["n"] == 0, a[k], torch.where(a["n"] == 0, b[k], r[k]))
    return r


def block_moments_ref(tab):
    """(moments with bounds of the channel's block merge, depth, CH): the warps merged as the 5-level shuffle tree."""
    c = tab.shape[2]
    ch = stats_group_channels(c)
    r, depth = _warp_moments(tab, ch)
    for o in (16, 8, 4, 2, 1):   # lane i merges lane i + o
        a = {k: v[:o] for k, v in r.items()}
        b = {k: v[o:2 * o] for k, v in r.items()}
        m = _merge_bound(a, b)
        r = {k: torch.cat([m[k], r[k][o:]]) for k in r}
    return {k: v[0] for k, v in r.items()}, depth + 5, ch


def finalize_ref(mo, gamma, beta, rm, rv):
    """finalize_channel in float64 with bounds. var = m2/n; invstd = rsqrtf(var + eps) (rsqrtf: <= 2 ulp = 4u);
    sc = gamma*invstd; sh = beta - mean*sc; running stats: nn.BatchNorm's update (1 - m)*r + m*v with the unbiased
    variance (the biased one at n = 1), three roundings + the rounding of 1 - m."""
    n, mean, m2, em, e2 = mo["n"], mo["mean"], mo["m2"], mo["em"], mo["e2"]
    c = n.numel()
    g = gamma.double() if gamma is not None else torch.ones(c, device="cuda", dtype=torch.float64)
    bt = beta.double() if beta is not None else torch.zeros(c, device="cuda", dtype=torch.float64)
    var = torch.where(n > 0, m2 / n.clamp_min(1), 0.0)
    ev = torch.where(n > 0, e2 / n.clamp_min(1), 0.0) + U * var
    v = var + EPS
    inv = v.rsqrt()
    einv = inv * (0.51 * (ev + U * v) / v + 5 * U)
    sc = g * inv
    esc = g.abs() * einv + U * sc.abs()
    sh = bt - mean * sc
    esh = sc.abs() * em + mean.abs() * esc + 2 * U * ((mean * sc).abs() + sh.abs())
    out = dict(mean=(mean, em), invstd=(inv, einv), count=(n, torch.zeros_like(n)), scale=(sc, esc),
               shift=(sh, esh))
    if rm is not None:
        r0 = rm.double()
        new = (1 - MOM) * r0 + MOM * mean
        out["running_mean"] = (new, 4 * U * ((1 - MOM) * r0.abs() + MOM * mean.abs()) + MOM * em)
        unb = torch.where(n > 1, m2 / (n - 1).clamp_min(1), var)
        eunb = torch.where(n > 1, e2 / (n - 1).clamp_min(1) + U * unb, ev)
        r1 = rv.double()
        out["running_var"] = ((1 - MOM) * r1 + MOM * unb, 4 * U * ((1 - MOM) * r1.abs() + MOM * unb) + MOM * eunb)
    return out


def finalize_outputs(mi, ss, rm, rv):
    got = dict(mean=mi[0], invstd=mi[1], count=mi[2], scale=ss[0], shift=ss[1])
    if rm is not None:
        got.update(running_mean=rm, running_var=rv)
    return got


def check_finalize(got, ref):
    """(worst ratio, worst key) over every output."""
    worst, key = 0.0, None
    for k, (r, b) in ref.items():
        w = worst_ratio(got[k], r, b)
        if w > worst:
            worst, key = w, k
    return worst, key


# id: (T rows, C, what the case guards)
FINALIZE = {
    "t1-c8": (1, 8, "a single row"),
    "t528-c72": (528, 72, "4 rows x 132 SMs (conv epilogue), CH 8, a partial block of one block"),
    "t2048-c8": (2048, 8, "CH 8: 16 rows per lane, the outer row loop runs twice (T > RL*U = 1024)"),
    "t528-c1032": (528, 1032, "CH 16, partial last block (1032 % 16 = 8)"),
    "t2048-c2048": (2048, 2048, "CH 16, 2048 rows (the bf16x3 K-slice finish maximum)"),
    "t2048-c2056": (2048, 2056, "CH 32, partial last block (2056 % 32 = 8)"),
    "t1-c2056": (1, 2056, "CH 32, a single row"),
}


@pytest.mark.parametrize("name", list(FINALIZE))
def test_finalize_partials_synthetic_tables(name):
    from semseg_b200 import ops
    t, c, what = FINALIZE[name]
    gen = torch.Generator(device="cuda").manual_seed(t * 7 + c)
    tab, ratios = synthetic_table(t, c, gen)
    gamma = torch.rand((c,), device="cuda", generator=gen) + 0.5
    beta = torch.randn((c,), device="cuda", generator=gen)
    rm0 = torch.randn((c,), device="cuda", generator=gen)
    rv0 = torch.rand((c,), device="cuda", generator=gen) + 0.5
    ch = stats_group_channels(c)
    claims = [what, "CH %d, %d blocks" % (ch, cdiv(c, ch))]
    assert ch == {8: 8, 72: 8, 1032: 16, 2048: 16, 2056: 32}[c]
    if name == "t2048-c8":
        assert cdiv(t, 1024 // ch) > 8, "more rows per lane than U = 8: the outer row loop runs more than once"
    if c % ch:
        claims.append("last block holds %d of %d channels" % (c % ch, ch))
    zero_rows = int((tab[:, 2, 0] == 0).sum())
    claims.append("%d zero-count rows" % zero_rows)
    tab0 = tab.clone()

    def run():
        rm, rv = rm0.clone(), rv0.clone()
        mi, ss = ops.bn_finalize_partials(tab, gamma, beta, EPS, MOM, rm, rv)
        return mi.clone(), ss.clone(), rm, rv

    mi, ss, rm, rv = run()
    mi2, ss2, rm2, rv2 = run()
    assert torch.equal(mi, mi2) and torch.equal(ss, ss2) and torch.equal(rm, rm2) and torch.equal(rv, rv2)
    assert torch.equal(tab, tab0), "the table was modified"
    mo, depth, _ = block_moments_ref(tab)
    ref = finalize_ref(mo, gamma, beta, rm0, rv0)
    got = finalize_outputs(mi, ss, rm, rv)
    assert torch.equal(mi[2].double(), tab.double()[:, 2].sum(0)), "count is not the exact sum of the row counts"
    worst, key = check_finalize(got, ref)
    # the merge alone (bn_merge_partials: the same block function): (mean, M2, n)
    mp = ops.bn_merge_partials(tab)
    mworst = max(worst_ratio(mp[0], mo["mean"], mo["em"]), worst_ratio(mp[1], mo["m2"], mo["e2"]))
    assert torch.equal(mp[2], mi[2])
    # measured relative variance error by mean/std ratio (the raw-moment form's weak spot)
    var_ref = mo["m2"] / mo["n"]
    rel = ((mp[1].double() / mp[2].double() - var_ref).abs() / var_ref).cpu()
    for rt in (0.0, 1.0, 30.0):
        sel = ratios == rt
        claims.append("mean/std %g: var rel err %.2g (bound %.2g)" %
                      (rt, float(rel[sel].max()), float((mo["e2"] / mo["m2"]).cpu()[sel].max())))
    claims.append("merge worst %.3g, finalise worst %.3g (%s)" % (mworst, worst, key))
    # teeth: the last row of the table left out
    tmo, _, _ = block_moments_ref(tab[:-1]) if t > 1 else (
        {k: torch.zeros_like(v) for k, v in mo.items()}, 0, 0)
    teeth = check_finalize(got, {k: (finalize_ref(tmo, gamma, beta, rm0, rv0)[k][0], ref[k][1]) for k in ref})[0]
    claims.append("teeth: last table row dropped")
    report("finalize-" + name, claims, max(worst, mworst), teeth)


@pytest.mark.parametrize("split", [False, True], ids=["bf16", "x3"])
def test_finalize_real_partials_from_conv(split):
    """Partials as the convolutions make them: the conv epilogue's per-warp rows (bf16 and bf16x3 without K slicing),
    and bf16x3's K-slice finish with 2048 chunk rows (3x3 conv, Cin 64: 9 K blocks, 2 slices; 512x512 pixels)."""
    from semseg_b200 import ops, _lib as L
    gen = torch.Generator(device="cuda").manual_seed(11 + split)
    cases = [(2, 40, 45, 64, 192, 1)]
    if split:
        cases.append((1, 512, 512, 64, 64, 3))
    claims, worst, teeth = [], 0.0, 0.0
    for n, h, w, cin, cout, k in cases:
        x = _act(torch.randn((n, h, w, cin), device="cuda", generator=gen) + 3.0, split)
        wt = torch.randn((cout, cin, k, k), device="cuda", generator=gen) / (cin * k * k) ** 0.5
        pw = ops.pack_weights(wt, split=split)
        _, sp = ops.conv_fprop(x, pw.wf, cout, ops.conv_taps(k, 1), stats=True)
        m = n * h * w
        if k == 3:
            assert sp.shape[0] == int(L.load().semseg_conv_splitk_rows(m)) == 2048, "K-slice finish: 2048 chunk rows"
            claims.append("K-slice finish: %d rows of %d pixels" % (sp.shape[0], m // sp.shape[0]))
        else:
            claims.append("conv epilogue: %d rows" % sp.shape[0])
        gamma = torch.rand((cout,), device="cuda", generator=gen) + 0.5
        beta = torch.randn((cout,), device="cuda", generator=gen)
        rm0, rv0 = torch.zeros(cout, device="cuda"), torch.ones(cout, device="cuda")
        rm, rv = rm0.clone(), rv0.clone()
        mi, ss = ops.bn_finalize_partials(sp, gamma, beta, EPS, MOM, rm, rv)
        assert bool((mi[2] == m).all())
        mo, _, _ = block_moments_ref(sp)
        got = finalize_outputs(mi, ss, rm, rv)
        wv, key = check_finalize(got, finalize_ref(mo, gamma, beta, rm0, rv0))
        last = sp[:-1] if bool((sp[-1, 2] > 0).all()) else sp[:int((sp[:, 2, 0] > 0).nonzero().max())]
        tmo, _, _ = block_moments_ref(last)
        tref = finalize_ref(tmo, gamma, beta, rm0, rv0)
        ref = finalize_ref(mo, gamma, beta, rm0, rv0)
        teeth = max(teeth, check_finalize(got, {kk: (tref[kk][0], ref[kk][1]) for kk in ref})[0])
        worst = max(worst, wv)
        claims.append("worst %.3g (%s)" % (wv, key))
    claims.append("teeth: last non-empty row dropped")
    report("finalize-conv-%s" % ("x3" if split else "bf16"), claims, worst, teeth)


@pytest.mark.parametrize("ranks", [1, 2, 3, 8])
def test_finalize_nccl_form(ranks):
    """bn_finalize over R gathered [3][C] blocks (each one rank's bn_merge_partials), merged in rank order, against
    the pooled float64 moments. Rank 0 (of R > 1) has no samples. R = 1: bit-identical to bn_finalize_partials (every
    finalise ends in finalize_channel, so equal moments give equal bits)."""
    from semseg_b200 import ops
    gen = torch.Generator(device="cuda").manual_seed(100 + ranks)
    c = 72
    tabs = [synthetic_table(t, c, gen)[0] for t in ([528] if ranks == 1 else [528, 1, 37, 2048, 5, 300, 528, 64][:ranks])]
    if ranks > 1:
        tabs[0] = tabs[0] * 0                     # a rank whose statistics count is 0
    gamma = torch.rand((c,), device="cuda", generator=gen) + 0.5
    beta = torch.randn((c,), device="cuda", generator=gen)
    rm0 = torch.randn((c,), device="cuda", generator=gen)
    rv0 = torch.rand((c,), device="cuda", generator=gen) + 0.5
    blocks = torch.stack([ops.bn_merge_partials(tb) for tb in tabs]).contiguous()
    rm, rv = rm0.clone(), rv0.clone()
    mi, ss = ops.bn_finalize(blocks, gamma, beta, EPS, MOM, rm, rv)
    acc = None
    for tb in tabs:
        mo, _, _ = block_moments_ref(tb)
        acc = mo if acc is None else _merge_bound(acc, mo)
    # the pooled float64 moments equal the merged reference to float64 rounding
    pooled = torch.cat(tabs).double()
    n_all = pooled[:, 2].sum(0)
    assert torch.equal(acc["n"], n_all)
    assert float(((acc["mean"] - pooled[:, 0].sum(0) / n_all).abs()).max()) <= 1e-9 * float(acc["mean"].abs().max())
    ref = finalize_ref(acc, gamma, beta, rm0, rv0)
    worst, key = check_finalize(finalize_outputs(mi, ss, rm, rv), ref)
    claims = ["%d ranks, counts %s" % (ranks, [int(tb[:, 2, 0].sum()) for tb in tabs]), "worst %s" % key]
    # teeth: the last rank's block left out
    tacc = None
    for tb in tabs[:-1] if ranks > 1 else [tabs[0][:-1]]:
        mo, _, _ = block_moments_ref(tb)
        tacc = mo if tacc is None else _merge_bound(tacc, mo)
    tref = finalize_ref(tacc, gamma, beta, rm0, rv0)
    teeth = check_finalize(finalize_outputs(mi, ss, rm, rv), {k: (tref[k][0], ref[k][1]) for k in ref})[0]
    claims.append("teeth: last %s dropped" % ("rank" if ranks > 1 else "table row"))
    if ranks == 1:
        rm2, rv2 = rm0.clone(), rv0.clone()
        mi2, ss2 = ops.bn_finalize_partials(tabs[0], gamma, beta, EPS, MOM, rm2, rv2)
        assert torch.equal(mi, mi2) and torch.equal(ss, ss2) and torch.equal(rm, rm2) and torch.equal(rv, rv2)
        claims.append("bit-identical to bn_finalize_partials")
    report("finalize-nccl-R%d" % ranks, claims, worst, teeth)


@pytest.mark.parametrize("split", [False, True], ids=["bf16", "x3"])
def test_finalize_one_pixel(split):
    """M = 1 (PPM bin 1 with one image per GPU), on the real conv partials of a 1x1 map: mean = the stored value,
    count 1, and the running variance takes the biased variance (there is no unbiased one). bf16: y^2 is exact in fp32,
    so M2 = Q - S*mean = 0, invstd = rsqrt(eps) and running_var = (1 - momentum) * running_var bit for bit. bf16x3:
    y has 16 significant bits, so M2 is at most the fp32 rounding of y^2 (2^-24 y^2). torch's BatchNorm raises here
    instead."""
    from semseg_b200 import ops
    gen = torch.Generator(device="cuda").manual_seed(1)
    c = 512
    x = _act(torch.randn((1, 1, 1, 2048), device="cuda", generator=gen), split)
    pw = ops.pack_weights(torch.randn((c, 2048, 1, 1), device="cuda", generator=gen) * 0.02, split=split)
    y, sp = ops.conv_fprop(x, pw.wf, c, ops.conv_taps(1, 1), stats=True)
    rm0 = torch.randn((c,), device="cuda", generator=gen)
    rv0 = torch.rand((c,), device="cuda", generator=gen) + 0.5
    rm, rv = rm0.clone(), rv0.clone()
    mi, ss = ops.bn_finalize_partials(sp, None, None, EPS, MOM, rm, rv)
    mp = ops.bn_merge_partials(sp)
    yv = pixels(y)[0]
    assert bool((mi[2] == 1).all())
    assert torch.equal(mi[0].double(), yv), "mean of one pixel is its stored value"
    if split:
        assert bool((mp[1].double() <= U * yv * yv).all()), "M2 beyond the rounding of y^2"
    else:
        assert bool((mp[1] == 0).all()), "M2 of one bf16 pixel is 0"
        inv = torch.tensor(EPS, dtype=torch.float64).rsqrt().item()
        assert float((mi[1].double() - inv).abs().max()) <= 4 * U * inv, "invstd = rsqrt(eps) within rsqrtf's 2 ulp"
        assert torch.equal(rv, (1 - torch.tensor(MOM, device="cuda")) * rv0), "running_var = (1 - m) * running_var"
    with pytest.raises(ValueError):
        torch.nn.functional.batch_norm(torch.zeros((1, c, 1, 1)), None, None, training=True)
    mo, _, _ = block_moments_ref(sp)
    worst, key = check_finalize(finalize_outputs(mi, ss, rm, rv), finalize_ref(mo, None, None, rm0, rv0))
    # teeth: a count off by one (n = 2: the unbiased running variance would be used and the mean halved)
    mo2 = dict(mo, n=mo["n"] + 1)
    tref = finalize_ref(mo2, None, None, rm0, rv0)
    ref = finalize_ref(mo, None, None, rm0, rv0)
    teeth = check_finalize(finalize_outputs(mi, ss, rm, rv), {k: (tref[k][0], ref[k][1]) for k in ref})[0]
    report("finalize-m1-%s" % ("x3" if split else "bf16"), ["%d rows, one with count 1" % sp.shape[0],
           "worst %s" % key, "teeth: count off by one"], worst, teeth)


# ------------------------------------------------------------------------------------------------ apply
# id: (M, C, options). xs / rs / os: (channel offset, buffer width) of x / residual / out inside a wider buffer.
APPLY = {
    "m1-c8-res-relu": (1, 8, dict(res=True, relu=True, teeth="pixel")),
    "m31-c72-slices-res-relu": (31, 72, dict(res=True, relu=True, xs=(16, 160), rs=(8, 88), os=(72, 152),
                                             teeth="res")),
    "m257-c256-plain": (257, 256, dict(teeth="group")),
    "m257-c256-relu": (257, 256, dict(relu=True, teeth="relu")),
    "m7200-c72-slices-relu": (7200, 72, dict(relu=True, xs=(8, 88), os=(0, 80), teeth="group")),
    "m7200-c2048-res-relu-multipass": (7200, 2048, dict(res=True, relu=True, teeth="pixel")),
}


@pytest.mark.parametrize("split", [False, True], ids=["bf16", "x3"])
@pytest.mark.parametrize("name", list(APPLY))
def test_bn_apply_element_bound(name, split):
    from semseg_b200 import ops
    m, c, o = APPLY[name]
    gen = torch.Generator(device="cuda").manual_seed(m * 13 + c)
    _, x = in_buffer(m, c, split, gen, *(o.get("xs") or (None, None)), scale=2.0, shift=0.5)
    res = in_buffer(m, c, split, gen, *o["rs"])[1] if "rs" in o else (
        in_buffer(m, c, split, gen)[1] if o.get("res") else None)
    ooff, owidth = o.get("os") or (None, None)
    obuf, out = out_buffer(m, c, split, ooff, owidth)
    _, ss, _, _ = coefficients(x, gen)
    relu = bool(o.get("relu"))
    claims = []
    for label, t in (("x", x), ("residual", res), ("out", out)):
        if t is not None and ops._nhwc_meta(t)[4] > c:
            claims.append("%s pitch %d > C" % (label, ops._nhwc_meta(t)[4]))
    pstride, passes, tail = stride_passes(m, c, 4)
    claims.append("pixel stride %d, %d pass(es)%s" % (pstride, passes, ", unroll tail" if tail else ""))
    if name.endswith("multipass"):
        assert m * c // 8 > _sms() * 16 * 256 and passes > 1, "the grid-stride loop runs more than once"
        assert tail, "some thread runs the non-unrolled tail"
    inputs = [t.clone() for t in (x, res, ss) if t is not None]
    ops.bn_apply(x, ss, residual=res, relu=relu, out=out)
    y1 = obuf.clone()
    ops.bn_apply(x, ss, residual=res, relu=relu, out=out)
    assert torch.equal(obuf, y1), "not bit-identical on a second call"
    assert all(torch.equal(a, b) for a, b in zip(inputs, [t for t in (x, res, ss) if t is not None]))
    assert_outside_untouched(obuf, ooff, c)

    # y = fmaf(x, sc, sh) + r, then fmaxf(., 0): two roundings, 2u*(|x*sc| + |sh| + |r|); ReLU is 1-Lipschitz
    xv, sc, sh = pixels(x), ss[0].double(), ss[1].double()
    rv = pixels(res) if res is not None else torch.zeros_like(xv)
    s = (xv * sc).abs() + sh.abs() + rv.abs()

    def ref_of(with_res=True, with_relu=relu):
        v = xv * sc + sh + (rv if with_res else 0)
        return v.clamp_min(0) if with_relu else v

    ref = ref_of()
    outv = pixels(out).reshape(1, 1, m, c)
    worst = act_ratio(out, ref.reshape(1, 1, m, c), s.reshape(1, 1, m, c), 2, split)
    t = o["teeth"]
    tref = ref.clone()
    if t == "pixel":
        tref[-1] = 0
        claims.append("teeth: last pixel not stored")
    elif t == "group":
        tref[:, c - 8:] = 0
        claims.append("teeth: last 8-channel group not stored")
    elif t == "res":
        tref = ref_of(with_res=False)
        claims.append("teeth: residual not added")
    else:
        tref = ref_of(with_relu=False)
        claims.append("teeth: ReLU not applied")
    teeth = ratio(outv, tref.reshape(1, 1, m, c), s.reshape(1, 1, m, c), R_SPLIT if split else R_BF16, 2)
    report("apply-%s-%s" % (name, "x3" if split else "bf16"), claims, worst, teeth)


# ------------------------------------------------------------------------------------------------ backward
# id: (M, C, options). relu: run the mask from y and from raw (bit-identical) or no ReLU. xs: x / dy / y as slices.
BWD = {
    "m2-c256-relu": (2, 256, dict(relu=True, teeth="pixel")),
    "m257-c72-relu-slices": (257, 72, dict(relu=True, slices=True, teeth="group")),
    "m257-c256-norelu": (257, 256, dict(relu=False, teeth="chunk")),
    "m7200-c2048-relu": (7200, 2048, dict(relu=True, teeth="relu")),
    "m7200-c72-norelu-slices": (7200, 72, dict(relu=False, slices=True, teeth="group")),
    "m80000-c72-relu-313-chunks": (80000, 72, dict(relu=True, teeth="chunk")),
}


def bwd_apply_raw(dy, y, x, mi, gamma, ss, sums, count, relu, dx, dres, dgb):
    """semseg_bn_bwd_apply through ctypes, so dx and dres can be channel slices (ops.bn_bwd_apply fixes their pitch)."""
    from semseg_b200 import ops, _lib as L
    lib = L.load()
    m = x.shape[-2] * x.shape[-3] * x.shape[-4]
    c = x.shape[-1]
    p = lambda t: ops._nhwc_meta(t)[4] if t is not None else 0      # noqa: E731
    L.check(lib.semseg_bn_bwd_apply(ops._ptr(dy), ops._lo(dy), p(dy), ops._ptr(y), ops._lo(y), p(y), ops._ptr(x),
                                    ops._lo(x), p(x), ops._ptr(mi), ops._ptr(gamma), ops._ptr(ss), ops._ptr(sums),
                                    float(count), m, c, int(relu), ops._ptr(dx), ops._lo(dx), p(dx), ops._ptr(dres),
                                    ops._lo(dres), p(dres), ops._ptr(dgb), ops._stream()), "semseg_bn_bwd_apply")


@pytest.mark.parametrize("split", [False, True], ids=["bf16", "x3"])
@pytest.mark.parametrize("name", list(BWD))
def test_bn_backward_element_bound(name, split):
    from semseg_b200 import ops, _lib as L
    m, c, o = BWD[name]
    relu = o["relu"]
    gen = torch.Generator(device="cuda").manual_seed(m * 17 + c)
    sl = o.get("slices")
    _, x = in_buffer(m, c, split, gen, *((8, c + 24) if sl else (None, None)), scale=2.0, shift=0.5)
    _, dy = in_buffer(m, c, split, gen, *((c + 16, 2 * c + 32) if sl else (None, None)))
    mi, ss, gamma, _ = coefficients(x, gen)
    y = None
    if relu:
        ybuf, y = out_buffer(m, c, split, *((16, c + 16) if sl else (None, None)))
        ops.bn_apply(x, ss, relu=True, out=y)
    rows, chunks = chunk_rows(m), cdiv(m, chunk_rows(m))
    unroll = 2 if split else 4
    last_rows = m - (chunks - 1) * rows
    claims = ["%d chunk(s) of %d rows, last %d" % (chunks, rows, last_rows)]
    if c % 64:
        claims.append("%d channel blocks, last with %d of 8 groups active" % (cdiv(c, 64), (c % 64) // 8))
        assert cdiv(c, 64) * 8 > c // 8, "inactive channel groups in the last block"
    if chunks > 256:
        claims.append("final reduce loops over %d chunks" % chunks)
    if name.endswith("313-chunks"):
        assert chunks == 313 > 32 * 8, "bn_bwd_reduce_final_kernel loops more than once"
    if last_rows % (unroll * 32) or rows % (unroll * 32):
        claims.append("unroll tail (%d rows in flight)" % unroll)
    if name == "m257-c72-relu-slices":
        assert last_rows % (unroll * 32), "the last chunk ends in the unroll tail"
    inputs = [t.clone() for t in (x, dy, y, mi, ss) if t is not None]

    # ---- reduce: mask from y, from raw (+ scale_shift), bit-identical
    sums_y, tot_y = ops.bn_bwd_reduce(dy, y, x, mi, relu, scale_shift=ss if relu else None)
    sums_y, tot_y = sums_y.clone(), tot_y.clone()
    assert torch.equal(sums_y, tot_y)
    again, _ = ops.bn_bwd_reduce(dy, y, x, mi, relu, scale_shift=ss if relu else None)
    assert torch.equal(again, sums_y), "not bit-identical on a second call"
    if relu:
        sums_x, _ = ops.bn_bwd_reduce(dy, None, x, mi, True, scale_shift=ss)
        assert torch.equal(sums_x, sums_y), "mask from raw + scale_shift != mask from y"
        claims.append("mask from y == mask from raw, bit for bit")
    # the single-rank form writes `sums` and leaves `sums_total` alone
    lib = L.load()
    ws, nf = ops.bn_workspace(m, c, "cuda")
    loc = torch.full((2, c), SENTINEL, device="cuda")
    tot = torch.full((2, c), SENTINEL, device="cuda")
    p = lambda t: ops._nhwc_meta(t)[4] if t is not None else 0      # noqa: E731
    L.check(lib.semseg_bn_bwd_reduce(ops._ptr(dy), ops._lo(dy), p(dy), ops._ptr(y), ops._lo(y), p(y), ops._ptr(x),
                                     ops._lo(x), p(x), ops._ptr(mi), ops._ptr(ss), m, c, int(relu), ops._ptr(ws), nf,
                                     ops._ptr(loc), ops._ptr(tot), None, 1, 0, 0, 0, None, ops._stream()),
            "semseg_bn_bwd_reduce")
    assert torch.equal(loc, sums_y) and bool((tot == SENTINEL).all())

    xv, dv = pixels(x), pixels(dy)
    mean, invstd = mi[0].double(), mi[1].double()
    mask = (xv * ss[0].double() + ss[1].double() > 0) if relu else torch.ones_like(xv, dtype=torch.bool)
    dz = torch.where(mask, dv, 0.0)
    xhat = (xv - mean) * invstd

    def sums_ref(dz_, upto=m):
        return torch.stack([dz_[:upto].sum(0), (dz_ * xhat)[:upto].sum(0)])

    # a += d; b = fmaf(d, (x - mean) * invstd, b): per thread rows/32 rows, 32 lanes in shared memory, the chunks in
    # the final kernel (at most `chunks` non-zero adds per channel), + 3 roundings of the term
    depth = rows / 32 + 32 + chunks + 3
    sref = sums_ref(dz)
    sabs = torch.stack([dz.abs().sum(0), (dz * xhat).abs().sum(0)])
    rworst = worst_ratio(sums_y, sref, depth * U * sabs)
    t = o["teeth"]
    if t == "chunk":
        tsums = sums_ref(dz, (chunks - 1) * rows) if chunks > 1 else torch.zeros_like(sref)
    elif t == "pixel":
        tsums = sums_ref(dz, m - 1)
    elif t == "group":
        tsums = sref.clone()
        tsums[:, 64 * ((c - 1) // 64):] = 0
    else:
        tsums = sums_ref(dv)
    rteeth = worst_ratio(sums_y, tsums, depth * U * sabs)

    # ---- apply: dx = ka*dz + kx*x + kb with the kernel's sums and mean_invstd
    ybuf_in = ybuf.clone() if relu else None
    dxbuf, dx = out_buffer(m, c, split, *((8, c + 16) if sl else (None, None)))
    drbuf, dres = out_buffer(m, c, split, *((c, 2 * c + 8) if sl else (None, None)))
    dgb = torch.empty((2, c), device="cuda")
    results = []
    for src, count in (("y", m), ("y", 0), ("raw", m)):
        if src == "raw" and not relu:
            continue
        bwd_apply_raw(dy, y if src == "y" else None, x, mi, gamma, ss if relu else None, sums_y, count, relu, dx,
                      dres, dgb)
        results.append((dxbuf.clone(), drbuf.clone(), dgb.clone()))
    for r in results[1:]:
        assert all(torch.equal(a, b) for a, b in zip(r, results[0])), "count 0 / mask from raw differ"
    claims.append("bwd_apply: count M == count 0 (mean_invstd[2])%s, bit for bit" % (" == mask from raw" if relu else ""))
    assert_outside_untouched(dxbuf, 8 if sl else None, c)
    assert_outside_untouched(drbuf, c if sl else None, c)
    assert all(torch.equal(a, b) for a, b in zip(inputs, [t for t in (x, dy, y, mi, ss) if t is not None]))
    if relu:
        assert torch.equal(ybuf, ybuf_in)
    assert torch.equal(pixels(dres), dz), "dres is not the masked dy"
    assert torch.equal(dgb[0], sums_y[1]) and torch.equal(dgb[1], sums_y[0]), "dgamma_dbeta != swapped sums"

    g = gamma.double()
    s1, s2 = sums_y[0].double(), sums_y[1].double()
    ka = g * invstd
    kx = -ka * invstd * s2 / m
    kb = -ka * s1 / m - kx * mean
    # ka: 1 rounding; kx: 3 products + 1/count: 5u|kx|; kb: 4u|ka*s1/M| + 6u|kx*mean| + u|kb|; the two fmas:
    # u|kx*x + kb| + u|dx|. Collected: 2u|ka*dz| + 7u|kx*x| + 7u|ka*s1/M| + 9u|kx*mean|, inside 10u*(the sum).
    s = (ka * dz).abs() + (kx * xv).abs() + (ka * s1 / m).abs() + (kx * mean).abs()

    def dx_ref(dz_):
        return ka * dz_ + kx * xv + kb

    shape = (1, 1, m, c)
    aworst = act_ratio(dx, dx_ref(dz).reshape(shape), s.reshape(shape), 10, split)
    if t == "chunk":
        tdx = dx_ref(dz)
        tdx[(chunks - 1) * rows:] = 0
    elif t == "pixel":
        tdx = dx_ref(dz)
        tdx[-1] = 0
    elif t == "group":
        tdx = dx_ref(dz)
        tdx[:, c - 8:] = 0
    else:
        tdx = dx_ref(dv)
    ateeth = ratio(stored(dx), tdx.reshape(shape), s.reshape(shape), R_SPLIT if split else R_BF16, 10)
    claims.append("reduce worst %.3g teeth %.3g; apply worst %.3g teeth %.3g" % (rworst, rteeth, aworst, ateeth))
    claims.append("teeth: %s" % {"chunk": "last chunk dropped", "pixel": "last pixel dropped",
                                 "group": "last 64-channel block / 8-channel group dropped",
                                 "relu": "ReLU mask not applied"}[t])
    report("bwd-%s-%s" % (name, "x3" if split else "bf16"), claims, max(rworst, aworst), min(rteeth, ateeth))


# ------------------------------------------------------------------------------------------------ element-wise ops
def _split_ref(v, split):
    """torch restatement of act_st8: hi = bf16_rn(v), lo = bf16_rn(v - hi)."""
    hi = v.to(torch.bfloat16)
    if not split:
        return hi
    return torch.stack([hi, (v - hi.float()).to(torch.bfloat16)])


def _f32(t):
    """act_unpack: hi + lo in fp32."""
    return t[0].float() + t[1].float() if t.dim() == 5 else t.float()


@pytest.mark.parametrize("split", [False, True], ids=["bf16", "x3"])
@pytest.mark.parametrize("m,c", [(1, 8), (257, 72), (7200, 2048)])
def test_elementwise_ops_bit_exact(m, c, split):
    """add_act, scale_nc, f32_to_act (zero padding C..Cp) and act_to_f32 bit for bit against fp32 torch arithmetic and
    the hi/lo re-split, with pitched inputs and outputs and a sentinel outside every written slice."""
    from semseg_b200 import ops, _lib as L
    lib = L.load()
    gen = torch.Generator(device="cuda").manual_seed(m + c)
    _, a = in_buffer(m, c, split, gen, 8, c + 24)
    _, b = in_buffer(m, c, split, gen, c + 8, 2 * c + 8)
    obuf, out = out_buffer(m, c, split, 16, c + 32)
    a0, b0 = a.clone(), b.clone()
    ops.add_act(a, b, out=out)
    first = obuf.clone()
    ops.add_act(a, b, out=out)
    assert torch.equal(obuf, first) and torch.equal(a, a0) and torch.equal(b, b0)
    assert torch.equal(out, _split_ref(_f32(a) + _f32(b), split)), "add_act"
    assert_outside_untouched(obuf, 16, c)

    # scale_nc: N = 2 images of M pixels, per-(image, channel) factors
    xbuf = _act(torch.randn((2, 1, m, c + 16), device="cuda", generator=gen), split)
    xv = xbuf[..., 8:8 + c]
    scale = torch.rand((2, c), device="cuda", generator=gen) * 2
    sbuf = ops.empty_act((2, 1, m, c + 8), split, "cuda").fill_(SENTINEL)
    sout = sbuf[..., :c]
    L.check(lib.semseg_scale_nc(ops._ptr(xv), ops._lo(xv), c + 16, ops._ptr(scale), ops._ptr(sout), ops._lo(sout),
                                c + 8, 2, m, c, ops._stream()), "semseg_scale_nc")
    want = _split_ref(_f32(xv) * scale[:, None, None, :], split)
    assert torch.equal(sout, want), "scale_nc"
    assert_outside_untouched(sbuf, 0, c)
    assert torch.equal(ops.scale_nc(xv, scale), want)

    # f32_to_act: C' = C - 3 fp32 columns at pitch C + 5, out Cp = C channels at pitch C + 8, zero padded
    cf = c - 3 if c > 8 else 5
    fin = torch.randn((m, c + 5), device="cuda", generator=gen) * 3
    tbuf = ops.empty_act((1, 1, m, c + 8), split, "cuda").fill_(SENTINEL)
    tout = tbuf[..., 8:8 + c]
    L.check(lib.semseg_f32_to_act(ops._ptr(fin), c + 5, ops._ptr(tout), ops._lo(tout), c + 8, m, cf, c,
                                  ops._stream()), "semseg_f32_to_act")
    padded = torch.zeros((1, 1, m, c), device="cuda")
    padded[0, 0, :, :cf] = fin[:, :cf]
    assert torch.equal(tout, _split_ref(padded, split)), "f32_to_act"
    assert_outside_untouched(tbuf, 8, c)

    # act_to_f32: input slice, output at pitch C + 4 (fp32 scalar stores), sentinel around it
    fbuf = torch.full((m, c + 4), SENTINEL, device="cuda")
    L.check(lib.semseg_act_to_f32(ops._ptr(a), ops._lo(a), ops._nhwc_meta(a)[4], ops._ptr(fbuf), c + 4, m, c,
                                  ops._stream()), "semseg_act_to_f32")
    assert torch.equal(fbuf[:, :c], _f32(a).reshape(m, c)), "act_to_f32"
    assert bool((fbuf[:, c:] == SENTINEL).all())
    assert torch.equal(ops.act_to_f32(a).reshape(m, c), _f32(a).reshape(m, c))
    print("\n[elementwise-m%d-c%d-%s] add_act, scale_nc, f32_to_act (C %d -> Cp %d), act_to_f32: bit-exact, pitched, "
          "sentinels intact" % (m, c, "x3" if split else "bf16", cf, c))


# ------------------------------------------------------------------------------------------------ end to end
@pytest.mark.parametrize("split", [False, True], ids=["bf16", "x3"])
def test_bn_stage_vs_float64_autograd(split):
    """finalise -> apply (+ residual + ReLU) -> bwd_reduce -> bwd_apply against float64 autograd of
    F.batch_norm(training=True) + residual, ReLU, with the per-kernel bounds above composed: the statistics table
    (fp32 sums of x and x^2) and the finalise bound give the errors of mean and invstd, which enter y through
    x*sc + sh and dx through ka, xhat and the sums. The reference takes the kernel's ReLU mask (mask-matched): an element
    within the bound of 0 may fall either side."""
    import torch.nn.functional as F
    from semseg_b200 import ops
    m, c = 3000, 136
    gen = torch.Generator(device="cuda").manual_seed(42 + split)
    _, x = in_buffer(m, c, split, gen, scale=2.0, shift=3.0)
    _, res = in_buffer(m, c, split, gen)
    _, dy = in_buffer(m, c, split, gen)
    xv, rv, dv = pixels(x), pixels(res), pixels(dy)
    table = torch.stack([xv.sum(0), (xv * xv).sum(0), torch.full((c,), float(m), device="cuda",
                                                                 dtype=torch.float64)]).float()[None]
    gamma = torch.rand((c,), device="cuda", generator=gen) + 0.5
    beta = torch.randn((c,), device="cuda", generator=gen)
    mi, ss = ops.bn_finalize_partials(table, gamma, beta, EPS, MOM, None, None)
    y = ops.bn_apply(x, ss, residual=res, relu=True)
    sums, _ = ops.bn_bwd_reduce(dy, y, x, mi, True)
    dx, dres, dgb = ops.bn_bwd_apply(dy, y, x, mi, gamma, sums, float(m), True, want_dres=True)

    # statistics: the table's own fp32 rounding of the exact sums (u|S|, u*Q) on top of the finalise bound
    mo, _, _ = block_moments_ref(table)
    s_exact = xv.sum(0)
    mean_x = s_exact / m
    mo["em"] = mo["em"] + U * s_exact.abs() / m
    mo["e2"] = mo["e2"] + U * (xv * xv).sum(0) + 2 * U * (s_exact * mean_x).abs()
    mo["mean"], mo["m2"] = mean_x, ((xv - mean_x) ** 2).sum(0)
    fr = finalize_ref(mo, gamma, beta, None, None)
    (mean, em), (inv, einv), (sc, esc), (sh, esh) = fr["mean"], fr["invstd"], fr["scale"], fr["shift"]

    xr = xv.t().reshape(1, c, m, 1).clone().requires_grad_(True)
    rr = rv.t().reshape(1, c, m, 1).clone().requires_grad_(True)
    g64 = gamma.double().clone().requires_grad_(True)
    b64 = beta.double().clone().requires_grad_(True)
    pre = F.batch_norm(xr, None, None, g64, b64, True, 0.0, EPS) + rr
    mask = (pixels(y) > 0).t().reshape(1, c, m, 1)
    yref = pre * mask
    yref.backward(dv.t().reshape(1, c, m, 1))
    to_mc = lambda t: t.detach().reshape(c, m).t()     # noqa: E731
    ys = xv.abs() * esc + esh                            # statistics errors through x*sc + sh
    s_apply = (xv * sc).abs() + sh.abs() + rv.abs()
    yw = ratio(pixels(y), to_mc(yref), ys / (2 * U) + s_apply, R_SPLIT if split else R_BF16, 2)
    yt = ratio(pixels(y), to_mc(yref) - rv * to_mc(mask), ys / (2 * U) + s_apply, R_SPLIT if split else R_BF16, 2)

    dz = torch.where(to_mc(mask), dv, 0.0)
    xhat = (xv - mean) * inv
    exhat = em * inv + (xv - mean).abs() * einv
    rows, chunks = chunk_rows(m), cdiv(m, chunk_rows(m))
    depth = rows / 32 + 32 + chunks + 3
    s1, s2 = dz.sum(0), (dz * xhat).sum(0)
    es1 = depth * U * dz.abs().sum(0)
    es2 = depth * U * (dz * xhat).abs().sum(0) + (dz.abs() * exhat).sum(0)
    ka = gamma.double() * inv
    inner = dz - s1 / m - xhat * s2 / m
    edx = gamma.double() * einv * inner.abs() + ka.abs() * (es1 / m + exhat * s2.abs() / m + xhat.abs() * es2 / m)
    kx = -ka * inv * s2 / m
    s_bwd = (ka * dz).abs() + (kx * xv).abs() + (ka * s1 / m).abs() + (kx * mean).abs()
    dxw = ratio(pixels(dx), to_mc(xr.grad), edx / (10 * U) + s_bwd, R_SPLIT if split else R_BF16, 10)
    dxt = ratio(pixels(dx), to_mc(xr.grad) * 0.99, edx / (10 * U) + s_bwd, R_SPLIT if split else R_BF16, 10)
    assert torch.equal(pixels(dres), to_mc(rr.grad)), "dres is the masked dy"
    gw = max(worst_ratio(dgb[0], g64.grad, es2), worst_ratio(dgb[1], b64.grad, es1))
    report("stage-e2e-%s" % ("x3" if split else "bf16"),
           ["M %d, C %d, mean/std ~ 1.5" % (m, c), "y worst %.3g, dx worst %.3g, dgamma/dbeta worst %.3g" %
            (yw, dxw, gw), "teeth: y without the residual, dx scaled by 0.99"],
           max(yw, dxw, gw), min(yt, dxt))
