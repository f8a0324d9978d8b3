"""Oracle of the FP8 (e4m3) eval path (semseg_b200/fp8.py, csrc/fp8.cu, the e4m3 mode of csrc/conv_igemm.cu).

e4m3 rounding is torch's float8_e4m3fn cast (round to nearest even) after a clamp to +-448: the kernels' cvt.rn.satfinite
saturates, while torch alone turns values >= 480 into NaN. Every quantisation multiplies by qscale = 448 / amax in fp32
first, exactly as the kernels do. The fake-quant network restates oracle/torch_oracle.py's fp32 network with every FP8
conv's input and weight quantised and dequantised at the same scales."""
import numpy as np
import torch
import torch.nn.functional as F

from oracle.torch_oracle import Oracle

E4M3 = torch.float8_e4m3fn
MAX = 448.0


def e4m3(v):
    """fp32 tensor -> float8_e4m3fn, saturating (NaN stays NaN)."""
    return v.float().clamp(-MAX, MAX).to(E4M3)


def qscale_of(amax):
    """fp32 (qscale, dequantisation scale) of an amax (an all-zero tensor: 1, 1)."""
    a = np.float32(amax) if amax > 0 else np.float32(MAX)
    return np.float32(MAX) / a, a / np.float32(MAX)


def quantize(x, qscale):
    """bf16 / fp32 tensor -> e4m3 of x * qscale (fp32 product)."""
    return e4m3(x.float() * torch.tensor(np.float32(qscale), dtype=torch.float32, device=x.device))


def pack_weights(w):
    """fp32 OIHW -> (e4m3 slab [taps][Cout][Cin], fp32 dequantisation scales [Cout]) as semseg_fp8_pack_weights."""
    w = w.detach().float()
    cout, cin, k, _ = w.shape
    amax = w.abs().reshape(cout, -1).amax(1)
    amax = torch.where(amax > 0, amax, torch.full_like(amax, MAX))
    qs = torch.tensor(MAX, dtype=torch.float32, device=w.device) / amax
    q = e4m3(w * qs[:, None, None, None])
    slab = q.view(torch.uint8).reshape(cout, cin, k * k).permute(2, 0, 1).contiguous().view(E4M3)
    return slab, amax / MAX


def dequant_weights(w):
    """The weights the FP8 conv multiplies by, as fp64 OIHW: e4m3(w * qscale_c) * (amax_c / 448)."""
    slab, sw = pack_weights(w)
    cout, cin, k, _ = w.shape
    q = slab.float().permute(1, 2, 0).reshape(cout, cin, k, k).double()
    return q * sw.double()[:, None, None, None]


def e4m3_order(b):
    """Byte codes of e4m3 values (uint8 tensor) -> integers in value order (adjacent representable values differ by 1;
    +0 and -0 both map to 0)."""
    b = b.to(torch.int32)
    mag = b & 0x7F
    return torch.where((b & 0x80) != 0, -mag, mag)


class FakeQuantOracle(Oracle):
    """oracle/torch_oracle.py's network (fp32) with every conv named in `amax` ({conv name: input amax}) fed
    dequantised e4m3 operands: x -> e4m3(x * qscale) * s_x, w -> per-output-channel e4m3 weights."""

    def __init__(self, sd, amax, **kw):
        super().__init__(sd, **kw)
        self.amax = dict(amax)

    def conv(self, x, name, stride=1, padding=0, dilation=1):
        a = self.amax.get(name)
        if a is None:
            return super().conv(x, name, stride, padding, dilation)
        qs, sx = qscale_of(a)
        xq = quantize(x, qs).float() * float(sx)
        wq = dequant_weights(self.sd[name + '.weight']).float()
        return F.conv2d(xq, wq, self.sd.get(name + '.bias'), stride, padding, dilation)
