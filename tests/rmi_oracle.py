"""float64 statements of the RMI (+ BCE + cross-entropy) contract (include/semseg_b200.h, semseg_b200/losses.py
RMILoss), the checker of the RMI tests.

`rmi_contract` states the contract term by term (pooled maps, moment sums, the 9x9 algebra by Cholesky solves) and
`rmi_grad` its closed-form gradient; `rmi_algebra` is the part after pooling, so that a test can feed it the kernels'
own pooled maps. `rmi_literal` states the loss a second time the way the paper's released code writes it: shifted views
of the pooled maps, torch.linalg.inv, torch.linalg.cholesky, and autograd for the gradient."""
import torch
import torch.nn.functional as F

from tests.dice_oracle import upsampled

CLIP = 1e-6


def _valid(target, c, ignore_index):
    return (target != ignore_index) & (target >= 0) & (target < c)


def _maps(z, target, ignore_index):
    """-> valid [N,H,W] bool, one-hot y [N,C,H,W], sigmoid s, q = s v + clip (float64)."""
    c = z.shape[1]
    valid = _valid(target, c, ignore_index)
    t = torch.where(valid, target, torch.zeros_like(target))
    vm = valid.unsqueeze(1).double()
    y = (torch.arange(c, device=z.device).view(1, c, 1, 1) == t.unsqueeze(1)).double() * vm
    s = torch.sigmoid(z)
    return valid, y, s, s * vm + CLIP


def _neigh(m):
    """[N,C,Hp,Wp] -> the 3x3 neighbourhood vectors [N,C,9,K], (dy, dx) row-major, cells row-major."""
    n, c, hp, wp = m.shape
    return F.unfold(m.reshape(n * c, 1, hp, wp), 3).reshape(n, c, 9, -1)


def rmi_algebra(Y, Q, alpha):
    """Pooled maps Y, Q [N,C,Hp,Wp] -> dict of float64 results: raw moment sums `mom` [N,C,189] in the kernels' order
    (sum a, sum b, a a' upper triangle, b b' upper triangle, a b'), r [N,C], the table T [N,C,9,18] = [G_ab' | 2 G_bb],
    the means ma, mb [N,C,9], the centred neighbourhoods at, bt [N,C,9,K], and dQ = dr/dQ [N,C,Hp,Wp]."""
    Y, Q = Y.double(), Q.double()
    a, b = _neigh(Y), _neigh(Q)
    kk = a.shape[-1]
    iu = torch.triu_indices(9, 9)
    raw_aa, raw_bb, raw_ab = a @ a.transpose(-1, -2), b @ b.transpose(-1, -2), a @ b.transpose(-1, -2)
    mom = torch.cat([a.sum(-1), b.sum(-1), raw_aa[..., iu[0], iu[1]], raw_bb[..., iu[0], iu[1]],
                     raw_ab.flatten(-2)], -1)
    ma, mb = a.mean(-1), b.mean(-1)
    at, bt = a - ma.unsqueeze(-1), b - mb.unsqueeze(-1)
    saa, sbb, sab = at @ at.transpose(-1, -2), bt @ bt.transpose(-1, -2), at @ bt.transpose(-1, -2)
    eye = torch.eye(9, dtype=torch.float64, device=Q.device)
    lp = torch.linalg.cholesky(sbb + alpha * eye)
    x = torch.cholesky_solve(sab.transpose(-1, -2), lp).transpose(-1, -2)       # S_ab P^-1
    am = saa - x @ sab.transpose(-1, -2) + alpha * eye
    am = 0.5 * (am + am.transpose(-1, -2))
    la = torch.linalg.cholesky(am)
    r = torch.log(torch.diagonal(la, dim1=-2, dim2=-1)).sum(-1)
    mx = torch.cholesky_solve(x, la)                                          # M X
    g_ab = -mx
    g_bb = 0.5 * x.transpose(-1, -2) @ mx
    T = torch.cat([g_ab.transpose(-1, -2), 2 * g_bb], -1)
    db = g_ab.transpose(-1, -2) @ at + 2 * g_bb @ bt                           # dr/db_k [N,C,9,K]
    n, c, hp, wp = Q.shape
    dq = F.fold(db.reshape(n * c, 9, kk), (hp, wp), 3).reshape(n, c, hp, wp)
    return dict(mom=mom, r=r, T=T, ma=ma, mb=mb, at=at, bt=bt, dQ=dq, K=kk)


def rmi_contract(z, target, ignore_index=255, bce_weight=0.5, alpha=5e-4, ce_weight=0.0):
    """Upsampled logits z [N,C,H,W] (float64), target [N,H,W] -> dict: loss, bce, rmi, ce, nv, Y, Q and rmi_algebra's
    results."""
    z = z.double()
    n, c, h, w = z.shape
    valid, y, s, q = _maps(z, target, ignore_index)
    vm = valid.unsqueeze(1).double()
    nv = int(valid.sum())
    bce = (vm * (F.softplus(z) - y * z)).sum() / (nv + 1)
    Y, Q = F.avg_pool2d(y, 4, 4), F.avg_pool2d(q, 4, 4)
    alg = rmi_algebra(Y, Q, alpha)
    rmi = alg["r"].sum() / (9 * n)
    ce = torch.zeros((), dtype=torch.float64)
    if nv > 0:
        t = torch.where(valid, target, torch.zeros_like(target))
        nll = -torch.log_softmax(z, 1).gather(1, t.unsqueeze(1)).squeeze(1)
        ce = (nll * valid).sum() / nv
    loss = bce_weight * bce + (1 - bce_weight) * rmi + ce_weight * ce
    return dict(loss=loss, bce=bce, rmi=rmi, ce=ce, nv=nv, Y=Y, Q=Q, **alg)


def rmi_grad(z, target, ignore_index=255, bce_weight=0.5, alpha=5e-4, ce_weight=0.0, res=None):
    """Closed-form d loss / d z (float64 [N,C,H,W]) of rmi_contract:

        (1-bce_weight)/(9N) [pooled] v s(1-s)/16 dr/dQ[cell] + bce_weight v (s - y)/(n_valid+1)
        + ce_weight v (softmax - y) / n_valid"""
    z = z.detach().double()
    n, c, h, w = z.shape
    res = rmi_contract(z, target, ignore_index, bce_weight, alpha, ce_weight) if res is None else res
    valid, y, s, _ = _maps(z, target, ignore_index)
    vm = valid.unsqueeze(1).double()
    nv = res["nv"]
    dq = res["dQ"].repeat_interleave(4, -2).repeat_interleave(4, -1)
    dq = F.pad(dq, (0, w - dq.shape[-1], 0, h - dq.shape[-2]))
    g = (1 - bce_weight) / (9 * n) * vm * s * (1 - s) / 16 * dq
    g = g + bce_weight * vm * (s - y) / (nv + 1)
    if nv > 0:
        g = g + ce_weight * vm * (torch.softmax(z, 1) - y) / nv
    return g


def rmi_grad_logits(logits_nhwc, zoom, dz):
    """The transpose of the align-corners upsample: d z [N,C,H,W] -> d logits, fp32-shaped NHWC [N,h,w,C] in float64."""
    x = logits_nhwc.detach().double().requires_grad_(True)
    zz = upsampled(x, zoom)
    (g,) = torch.autograd.grad(zz, x, dz)
    return g


def rmi_literal(z, target, ignore_index=255, bce_weight=0.5, alpha=5e-4, ce_weight=0.0):
    """The loss as the paper's code writes it (float64, differentiable in z): one-hot labels and sigmoid probabilities
    masked by the valid map, 4x4 average pooling, the 9 shifted views stacked into vectors, centred, covariances by
    matmul, torch.linalg.inv of the regularised prediction covariance, the approximate posterior variance, and
    1/2 log det by torch.linalg.cholesky; per-class mean over the batch divided by 9 and summed over classes. The maps
    are computed in z's dtype and the vectors cast to float64 before the algebra, as that code does; the result is
    float64."""
    n, c, h, w = z.shape
    valid = _valid(target, c, ignore_index)
    mask = valid.unsqueeze(1).to(z.dtype)
    t = torch.where(valid, target, torch.zeros_like(target))
    one_hot = F.one_hot(t, c).permute(0, 3, 1, 2).to(z.dtype) * mask
    bce = F.binary_cross_entropy_with_logits(z, one_hot, weight=mask.expand_as(z), reduction="sum")
    bce = bce / (mask.sum() + 1.0)
    probs = torch.sigmoid(z) * mask + CLIP
    la = F.avg_pool2d(one_hot, 4, 4)
    pr = F.avg_pool2d(probs, 4, 4)
    hp, wp = la.shape[-2:]
    nh, nw = hp - 2, wp - 2
    la_v = torch.stack([la[:, :, y:y + nh, x:x + nw] for y in range(3) for x in range(3)], 2).reshape(n, c, 9, -1)
    pr_v = torch.stack([pr[:, :, y:y + nh, x:x + nw] for y in range(3) for x in range(3)], 2).reshape(n, c, 9, -1)
    la_v, pr_v = la_v.double(), pr_v.double()
    la_v = la_v - la_v.mean(3, keepdim=True)
    pr_v = pr_v - pr_v.mean(3, keepdim=True)
    la_cov = la_v @ la_v.transpose(2, 3)
    pr_cov = pr_v @ pr_v.transpose(2, 3)
    la_pr_cov = la_v @ pr_v.transpose(2, 3)
    eye = torch.eye(9, dtype=torch.float64, device=z.device)
    pr_cov_inv = torch.linalg.inv(pr_cov + alpha * eye)
    appro_var = la_cov - la_pr_cov @ pr_cov_inv @ la_pr_cov.transpose(2, 3)
    chol = torch.linalg.cholesky(appro_var + alpha * eye)
    rmi_now = 0.5 * 2.0 * torch.log(torch.diagonal(chol, dim1=-2, dim2=-1)).sum(-1)
    rmi = (rmi_now.mean(0) / 9.0).sum()
    loss = bce_weight * bce.double() + (1 - bce_weight) * rmi
    nv = int(valid.sum())
    if ce_weight != 0.0 and nv > 0:
        tt = torch.where(valid, target, torch.full_like(target, -100))
        loss = loss + ce_weight * F.cross_entropy(z, tt, ignore_index=-100).double()
    return loss
