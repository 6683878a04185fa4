"""Float64 CPU reference of one SA module in training mode, from given ball-query indices: QueryAndGroup(use_xyz) rows,
[1x1 conv -> BatchNorm2d with batch statistics | conv + bias] -> ReLU per layer, max-pool over the samples, the running
statistics update, and the backward of all of it against an upstream gradient.

BatchNorm, ReLU and the max-pool are written as autograd Functions with explicit backward formulas so that the tests can
(a) evaluate the backward with another implementation's decisions (its ReLU masks and chosen samples) and (b) build the
mutants that show the tolerances catch real mistakes:
    no_sum_g         BN backward without the sum(g)/n term
    no_sum_gx        BN backward without the xhat * sum(g xhat)/n term
    unbiased_norm    normalise with the unbiased variance
    biased_running   running_var updated with the biased variance
    wrong_pool       max-pool gradient routed to the smallest sample instead of the largest
    no_relu_mask     ReLU backward passes the gradient unmasked
"""
import torch

MUTANTS = ("no_sum_g", "no_sum_gx", "unbiased_norm", "biased_running", "wrong_pool", "no_relu_mask")


def ball_query(radius, nsample, xyz, centres):
    """(B, P, nsample) int64: the first nsample points with d^2 < r^2 in index order, padded with the first hit (0 without one)"""
    B, P = centres.shape[:2]
    d2 = ((centres[:, :, None, :].double() - xyz[:, None, :, :].double()) ** 2).sum(-1)
    idx = torch.zeros((B, P, nsample), dtype=torch.long)
    for b in range(B):
        for p in range(P):
            hits = torch.nonzero(d2[b, p] < radius * radius).flatten()[:nsample]
            if len(hits):
                idx[b, p, :] = hits[0]
                idx[b, p, :len(hits)] = hits
    return idx


class _BN(torch.autograd.Function):
    @staticmethod
    def forward(ctx, z, gamma, beta, eps, mutant):
        n = z.shape[0]
        mean = z.mean(0)
        var = ((z - mean) ** 2).mean(0)
        var_norm = var * n / (n - 1) if mutant == "unbiased_norm" else var
        invstd = 1.0 / torch.sqrt(var_norm + eps)
        xhat = (z - mean) * invstd
        ctx.save_for_backward(xhat, invstd, gamma)
        ctx.mutant = mutant
        ctx.stats = (mean, var)
        return gamma * xhat + beta

    @staticmethod
    def backward(ctx, g):
        xhat, invstd, gamma = ctx.saved_tensors
        t = g.clone()
        if ctx.mutant != "no_sum_g":
            t = t - g.mean(0)
        if ctx.mutant != "no_sum_gx":
            t = t - xhat * (g * xhat).mean(0)
        return gamma * invstd * t, (g * xhat).sum(0), g.sum(0), None, None


class _ReLU(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, mask, mutant):
        m = (x > 0) if mask is None else mask
        ctx.save_for_backward(m)
        ctx.mutant = mutant
        return x * m

    @staticmethod
    def backward(ctx, g):
        (m,) = ctx.saved_tensors
        return (g if ctx.mutant == "no_relu_mask" else g * m), None, None


class _Pool(torch.autograd.Function):
    """y (G, ns, C) -> max over ns; the gradient goes to `route` (G, C)"""

    @staticmethod
    def forward(ctx, y, route):
        ctx.save_for_backward(route)
        ctx.shape = y.shape
        return y.max(1).values

    @staticmethod
    def backward(ctx, g):
        (route,) = ctx.saved_tensors
        d = torch.zeros(ctx.shape, dtype=g.dtype)
        d.scatter_(1, route.unsqueeze(1), g.unsqueeze(1))
        return d, None


def layer_params(mlp):
    """[dict(w, b, gamma, beta, rm, rv, nbt, eps, momentum)] of a SharedMLP, float64 CPU copies"""
    out = []
    for layer in mlp.children():
        conv = layer.conv
        d = dict(w=conv.weight.detach().double().cpu().flatten(1),
                 b=None if conv.bias is None else conv.bias.detach().double().cpu())
        if hasattr(layer, "bn"):
            bn = layer.bn.bn
            d.update(gamma=bn.weight.detach().double().cpu(), beta=bn.bias.detach().double().cpu(),
                     rm=bn.running_mean.detach().double().cpu(), rv=bn.running_var.detach().double().cpu(),
                     nbt=int(bn.num_batches_tracked), eps=bn.eps, momentum=bn.momentum)
        out.append(d)
    return out


def scale(xyz, centres, feats, idx, layers, grad_out=None, masks=None, chosen=None, mutant=None):
    """one scale.  xyz (B, N, 3), centres (B, P, 3), feats (B, C, N) or None, idx (B, P, ns); layers from layer_params.
    masks (per layer (rows, C_l) bool) / chosen ((B*P, C_last) int64): decisions to use instead of the reference's own.
    -> dict(out (B, C_last, P), pre [per layer (rows, C_l) pre-activation], running [(rm, rv, nbt)], and with grad_out
    (B, C_last, P) the gradients: w, b, gamma, beta (lists per layer, None where absent) and feats)"""
    xyz, centres = xyz.double().cpu(), centres.double().cpu()
    idx = idx.long().cpu()
    B, P, ns = idx.shape
    bi = torch.arange(B)[:, None, None]
    rel = xyz[bi, idx] - centres[:, :, None, :]                                    # (B, P, ns, 3)
    fleaf = None
    cols = [rel.reshape(-1, 3)]
    if feats is not None:
        fleaf = feats.detach().double().cpu().requires_grad_(grad_out is not None)
        cols.append(fleaf.transpose(1, 2)[bi, idx].reshape(-1, fleaf.shape[1]))
    a = torch.cat(cols, 1)
    leaves, pre, running = [], [], []
    for l, d in enumerate(layers):
        w = d["w"].clone().requires_grad_(True)
        b = None if d["b"] is None else d["b"].clone().requires_grad_(True)
        z = a @ w.t() + (b if b is not None else 0)
        if "gamma" in d:
            g_, be = d["gamma"].clone().requires_grad_(True), d["beta"].clone().requires_grad_(True)
            y = _BN.apply(z, g_, be, d["eps"], mutant)
            n = z.shape[0]
            mean, var = z.detach().mean(0), z.detach().var(0, unbiased=False)
            run_var = var if mutant == "biased_running" else var * n / (n - 1)
            m = d["momentum"]
            running.append(((1 - m) * d["rm"] + m * mean, (1 - m) * d["rv"] + m * run_var, d["nbt"] + 1))
        else:
            g_ = be = None
            y = z
        leaves.append((w, b, g_, be))
        pre.append(y.detach())
        a = _ReLU.apply(y, None if masks is None else masks[l].cpu(), mutant)
    C = a.shape[1]
    yg = a.view(B * P, ns, C)
    if chosen is None:
        route = yg.detach().argmin(1) if mutant == "wrong_pool" else yg.detach().argmax(1)
    else:
        route = chosen.long().cpu()
    out = _Pool.apply(yg, route).view(B, P, C).transpose(1, 2)
    res = dict(out=out.detach(), pre=pre, running=running)
    if grad_out is not None:
        out.backward(grad_out.double().cpu())
        res["w"] = [x[0].grad for x in leaves]
        res["b"] = [x[1].grad if x[1] is not None else None for x in leaves]
        res["gamma"] = [x[2].grad if x[2] is not None else None for x in leaves]
        res["beta"] = [x[3].grad if x[3] is not None else None for x in leaves]
        res["feats"] = None if fleaf is None else fleaf.grad
    return res


# tolerances of the device path against this reference (TF32 GEMMs with fp32 accumulation)
FWD_TOL = 2e-3          # max|d| <= FWD_TOL * max|ref|: outputs, running statistics
GRAD_TOL = 5e-3         # max|d| <= GRAD_TOL * max|ref| ...
FROB_TOL = 2e-3         # ... and |d|_F <= FROB_TOL * |ref|_F: gradients (with the device's decisions); 4 TF32 unit
                        # roundoffs (2^-11): a weight gradient passes through two TF32 GEMMs (dA of the layer above, dW)


def fwd_ratio(got, ref):
    """error over tolerance of a forward quantity (<= 1 passes)"""
    got, ref = got.double().cpu(), ref.double().cpu()
    return float((got - ref).abs().max() / (FWD_TOL * ref.abs().max().clamp_min(1e-30)))


def grad_ratio(got, ref):
    """error over tolerance of a gradient: the larger of the max-abs and the relative-Frobenius ratios (<= 1 passes)"""
    got, ref = got.double().cpu(), ref.double().cpu()
    d = got - ref
    return max(float(d.abs().max() / (GRAD_TOL * ref.abs().max().clamp_min(1e-30))),
               float(d.norm() / (FROB_TOL * ref.norm().clamp_min(1e-30))))


def all_ratios(got, ref):
    """{name: ratio} over every quantity two scale() results share"""
    out = {"out": fwd_ratio(got["out"], ref["out"])}
    for l, (a, b) in enumerate(zip(got["running"], ref["running"])):
        # a mean can cancel to far below its summands: its scale is the larger of itself and the running std
        d = (a[0].double().cpu() - b[0]).abs().max()
        out["running_mean%d" % l] = float(d / (FWD_TOL * torch.maximum(b[0].abs().max(), b[1].clamp_min(0).sqrt().max())))
        out["running_var%d" % l] = fwd_ratio(a[1], b[1])
    for k in ("w", "b", "gamma", "beta"):
        for l, (a, b) in enumerate(zip(got.get(k, []), ref.get(k, []))):
            if a is None or b is None:
                continue
            if k == "beta":
                # sum(g) cancels like a mean; sum(g xhat) (the gamma gradient) sums the same g at unit scale
                a, b, scale = a.double().cpu(), b.double().cpu(), ref["gamma"][l].abs().max()
                d = a - b
                out["beta%d" % l] = max(float(d.abs().max() / (GRAD_TOL * torch.maximum(b.abs().max(), scale))),
                                        float(d.norm() / (FROB_TOL * torch.maximum(b.norm(), ref["gamma"][l].norm()))))
            else:
                out["%s%d" % (k, l)] = grad_ratio(a, b)
    if got.get("feats") is not None and ref.get("feats") is not None:
        out["feats"] = grad_ratio(got["feats"], ref["feats"])
    return out
