"""GPU tier (-m gpu): the batch-statistics rows of the fprop/dgrad convolution's RAW epilogue, bit for bit.

The kernel keeps each statistics row's running (sum, sum of squares, count) in registers across a CTA's tiles and adds
them to the row in global memory when the CTA moves to another channel tile or runs out of items. Its contract is the
per-tile update it replaced: row g of CTA b is the fp32 sum, in the CTA's item order, of each tile's fp32 column sums
over that tile's valid pixel rows [32g, 32g + 32), taken in row order (sum of squares as fma), of the stored output
(hi + lo for bf16x3). The reference rebuilds exactly that from the kernel's own output, for every channel-tile width
(Cout 64 ... 2048), a partial last wave, a grid smaller than the SM count, boxes clipped by the right image edge (valid
rows not a prefix), and both storage forms; `torch.equal` on the whole buffer. Cout = 2048 on a 132-SM H100 has 8
channel tiles, so every CTA alternates between two of them (a flush per tile); Cout <= 1024 keeps one per CTA.
"""
import numpy as np
import pytest
import torch

from tests.test_conv_edges_gpu import _act, _sms, cdiv, choose_box, conv_block_n

pytestmark = pytest.mark.gpu

# (N, H, W, Cin, Cout, k). bf16x3 runs the cases with taps * ceil(Cin / 64) <= 8 K blocks: longer ones are K-sliced, and
# the K-slice finish, not this kernel, takes their statistics
CASES = {
    "cout64-partial-wave": (24, 29, 31, 64, 64, 3),
    "cout128-clipped": (8, 61, 67, 128, 128, 1),
    "cout256-1x1": (20, 30, 30, 256, 256, 1),
    "cout512-two-ntiles": (10, 30, 30, 128, 512, 1),
    "cout1024-four-ntiles": (8, 30, 30, 64, 1024, 1),
    "cout2048-alternating": (4, 30, 30, 256, 2048, 1),
    "cout2048-small-grid": (1, 9, 9, 64, 2048, 1),
    "cout192-small-grid": (1, 12, 10, 64, 192, 3),
}


def stats_reference(v, cout):
    """[grid*4][3][cout] fp32 rows from the output values v (float32 numpy [N,H,W,cout]), in the kernel's order."""
    n, h, w, _ = v.shape
    bh, bw = choose_box(h, w, 128)
    th, tw = cdiv(h, bh), cdiv(w, bw)
    bn = conv_block_n(cout)
    n_tiles = cdiv(cout, bn)
    items = n * th * tw * n_tiles
    grid = min(items, _sms())
    out = np.zeros((grid * 4, 3, cout), np.float32)
    for b in range(grid):
        for item in range(b, items, grid):
            m_tile, n_tile = divmod(item, n_tiles)
            img, rem = divmod(m_tile, th * tw)
            h0, w0 = (rem // tw) * bh, (rem % tw) * bw
            cols = slice(n_tile * bn, min(cout, (n_tile + 1) * bn))
            for g in range(4):
                s = np.zeros(cols.stop - cols.start, np.float32)
                q = np.zeros_like(s)
                cnt = 0
                for r in range(32 * g, 32 * g + 32):
                    hi, wi = divmod(r, bw)
                    if r >= bh * bw or h0 + hi >= h or w0 + wi >= w:
                        continue
                    f = v[img, h0 + hi, w0 + wi, cols]
                    s = s + f
                    q = (q.astype(np.float64) + f.astype(np.float64) ** 2).astype(np.float32)   # fmaf(f, f, q)
                    cnt += 1
                row = out[b * 4 + g]
                row[0, cols] += s
                row[1, cols] += q
                row[2, cols] += np.float32(cnt)
    return out


RUNS = [(name, False) for name in CASES] + [(name, True) for name, c in CASES.items()
                                            if c[5] ** 2 * cdiv(c[3], 64) <= 8]


@pytest.mark.parametrize("name,split", RUNS, ids=["%s-%s" % (n, "bf16x3" if s else "bf16") for n, s in RUNS])
def test_conv_stats_rows_bit_exact(name, split):
    from semseg_b200 import ops
    n, h, w, cin, cout, k = CASES[name]
    g = torch.Generator(device="cuda").manual_seed(7)
    x = _act(torch.randn((n, h, w, cin), device="cuda", generator=g), split)
    wt = torch.randn((cout, cin, k, k), device="cuda", generator=g) * (1.0 / (cin * k * k) ** 0.5)
    pw = ops.pack_weights(wt, need_dgrad=False, split=split)
    y, sp = ops.conv_fprop(x, pw.wf, cout, ops.conv_taps(k, 1), stats=True)
    torch.cuda.synchronize()
    v = (y[0].float() + y[1].float()) if split else y.float()
    ref = torch.from_numpy(stats_reference(v.cpu().numpy(), cout))
    assert sp.shape == ref.shape
    assert torch.equal(sp.cpu(), ref), "statistics rows differ from the per-tile update at %d elements" % int(
        (sp.cpu() != ref).sum())
    y2, sp2 = ops.conv_fprop(x, pw.wf, cout, ops.conv_taps(k, 1), stats=True)
    assert torch.equal(y2, y) and torch.equal(sp2, sp)
