"""float64 torch oracle of the relation term of losses.DistillationLoss (CIRKD's mini-batch pixel-to-pixel relation):
the definition in the class docstring, written as directly as possible, with its closed-form gradient.

Features are [B, h, w, C] (NHWC) float tensors. `round_nodes` rounds the normalised nodes to bf16 where the kernels do
(once, after the fp32 normalisation), with a straight-through gradient: the kernels differentiate the unrounded
normalisation."""
import torch


def pool_nodes(f, pool):
    """max_pool2d(kernel=pool, stride=pool, ceil_mode=True) per channel -> (x [B, M, C], idx [B, M, C]): idx is the
    flat h*w position of the first maximum in row-major window order, as torch's."""
    b, h, w, c = f.shape
    x, idx = torch.nn.functional.max_pool2d(f.permute(0, 3, 1, 2), pool, pool, ceil_mode=True, return_indices=True)
    return x.permute(0, 2, 3, 1).reshape(b, -1, c), idx.permute(0, 2, 3, 1).reshape(b, -1, c)


def normalise(x):
    """x / |x| per node; a node with |x| < 1e-12 is the zero vector (and, as x * 0, gets no gradient)."""
    n = x.norm(dim=-1, keepdim=True)
    inv = torch.where(n < 1e-12, torch.zeros_like(n), 1.0 / n.clamp_min(1e-12))
    return x * inv


def nodes(f, pool, round_nodes=False):
    xh = normalise(pool_nodes(f.double(), pool)[0])
    if round_nodes:
        xh = xh + (xh.to(torch.bfloat16).double() - xh).detach()
    return xh


def relation_loss_nodes(xs, xt, tau):
    """R of node sets [B, M, C] as the per-pair loop of the definition."""
    b, m, _ = xs.shape
    total = xs.new_zeros(())
    for i in range(b):
        for j in range(b):
            ls = torch.log_softmax(xs[i] @ xs[j].T / tau, dim=1)
            lt = torch.log_softmax(xt[i] @ xt[j].T / tau, dim=1)
            total = total + (lt.exp() * (lt - ls)).sum()
    return total * tau * tau / (b * b * m)


def relation_loss(fs, ft, tau, pool, round_nodes=False):
    return relation_loss_nodes(nodes(fs, pool, round_nodes), nodes(ft, pool, round_nodes).detach(), tau)


def relation_grad(fs, ft, tau, pool, round_nodes=False):
    """Closed-form dR/dfs: dR/d(X_i X_j^T) = tau/(B^2 M) (P - Q) for every ordered pair, through the normalisation
    (dx^ - x^ (x^ . dx^)) / |x| (0 for a zero node) and the first window maximum."""
    fs = fs.double()
    b, h, w, c = fs.shape
    x, idx = pool_nodes(fs, pool)
    n = x.norm(dim=-1, keepdim=True)
    inv = torch.where(n < 1e-12, torch.zeros_like(n), 1.0 / n.clamp_min(1e-12))
    xh = x * inv
    xs = xh.to(torch.bfloat16).double() if round_nodes else xh
    xt = nodes(ft, pool, round_nodes)
    m = xs.shape[1]
    dxs = torch.zeros_like(xs)
    for i in range(b):
        for j in range(b):
            p = torch.softmax(xs[i] @ xs[j].T / tau, dim=1)
            q = torch.softmax(xt[i] @ xt[j].T / tau, dim=1)
            g = (p - q) * (tau / (b * b * m))
            dxs[i] += g @ xs[j]
            dxs[j] += g.T @ xs[i]
    dx = (dxs - xh * (xh * dxs).sum(-1, keepdim=True)) * inv
    df = torch.zeros((b, c, h * w), dtype=torch.float64, device=fs.device)
    df.scatter_add_(2, idx.permute(0, 2, 1), dx.permute(0, 2, 1))
    return df.reshape(b, c, h, w).permute(0, 2, 3, 1)
