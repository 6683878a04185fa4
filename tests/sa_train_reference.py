"""Float64 reference (on the CPU unless asked otherwise) of one SA module in training mode, from given ball-query indices: QueryAndGroup(use_xyz) rows,
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
        d = torch.zeros(ctx.shape, dtype=g.dtype, device=g.device)
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


def rows0(xyz, centres, feats, idx, device="cpu"):
    """layer 0's input rows (B * P * ns, 3 + C) in float64: [xyz[idx] - centre | feats[idx]]"""
    xyz, centres, idx = xyz.double().to(device), centres.double().to(device), idx.long().to(device)
    bi = torch.arange(idx.shape[0], device=device)[:, None, None]
    cols = [(xyz[bi, idx] - centres[:, :, None, :]).reshape(-1, 3)]
    if feats is not None:
        cols.append(feats.detach().double().to(device).transpose(1, 2)[bi, idx].reshape(-1, feats.shape[1]))
    return torch.cat(cols, 1)


def scale(xyz, centres, feats, idx, layers, grad_out=None, masks=None, chosen=None, mutant=None, device="cpu"):
    """one scale.  xyz (B, N, 3), centres (B, P, 3), feats (B, C, N) or None, idx (B, P, ns); layers from layer_params.
    masks (per layer (rows, C_l) bool) / chosen ((B*P, C_last) int64): decisions to use instead of the reference's own.
    device: where the float64 evaluation runs (on integer-valued data it is exact in any summation order, so a GPU
    evaluation is the same answer as the CPU one).
    -> dict(out (B, C_last, P), pre [per layer (rows, C_l) pre-activation], running [(rm, rv, nbt)], and with grad_out
    (B, C_last, P) the gradients: w, b, gamma, beta (lists per layer, None where absent), feats, and dz [per layer the
    gradient of conv output + bias])"""
    xyz, centres = xyz.double().to(device), centres.double().to(device)
    idx = idx.long().to(device)
    B, P, ns = idx.shape
    bi = torch.arange(B, device=device)[:, None, None]
    rel = xyz[bi, idx] - centres[:, :, None, :]                                    # (B, P, ns, 3)
    fleaf = None
    cols = [rel.reshape(-1, 3)]
    if feats is not None:
        fleaf = feats.detach().double().to(device).requires_grad_(grad_out is not None)
        cols.append(fleaf.transpose(1, 2)[bi, idx].reshape(-1, fleaf.shape[1]))
    a = torch.cat(cols, 1)
    del rel, cols
    leaves, pre, running, zs = [], [], [], []
    for l, d in enumerate(layers):
        w = d["w"].to(device).clone().requires_grad_(True)
        b = None if d["b"] is None else d["b"].to(device).clone().requires_grad_(True)
        z = a @ w.t() + (b if b is not None else 0)
        if grad_out is not None:
            z.retain_grad()
        zs.append(z)
        if "gamma" in d:
            g_, be = d["gamma"].to(device).clone().requires_grad_(True), d["beta"].to(device).clone().requires_grad_(True)
            y = _BN.apply(z, g_, be, d["eps"], mutant)
            n = z.shape[0]
            mean, var = z.detach().mean(0), z.detach().var(0, unbiased=False)
            run_var = var if mutant == "biased_running" else var * n / (n - 1)
            m = d["momentum"]
            running.append(((1 - m) * d["rm"].to(device) + m * mean, (1 - m) * d["rv"].to(device) + m * run_var, d["nbt"] + 1))
        else:
            g_ = be = None
            y = z
        leaves.append((w, b, g_, be))
        pre.append(y.detach())
        a = _ReLU.apply(y, None if masks is None else masks[l].to(device), mutant)
    C = a.shape[1]
    yg = a.view(B * P, ns, C)
    if chosen is None:
        route = yg.detach().argmin(1) if mutant == "wrong_pool" else yg.detach().argmax(1)
    else:
        route = chosen.long().to(device)
    out = _Pool.apply(yg, route).view(B, P, C).transpose(1, 2)
    res = dict(out=out.detach(), pre=pre, running=running)
    if grad_out is not None:
        out.backward(grad_out.double().to(device))
        res["w"] = [x[0].grad for x in leaves]
        res["b"] = [x[1].grad if x[1] is not None else None for x in leaves]
        res["gamma"] = [x[2].grad if x[2] is not None else None for x in leaves]
        res["beta"] = [x[3].grad if x[3] is not None else None for x in leaves]
        res["feats"] = None if fleaf is None else fleaf.grad
        res["dz"] = [z.grad for z in zs]
    return res


# ---------------------------------------------------------------------------------------------- integer-valued cases
# With integer operands of at most 2048 in magnitude, every TF32 conversion is exact; with every partial sum below 2^24,
# every fp32 product and sum is exact in any order.  The device path then has exactly one right answer for Z, the
# outputs, the chosen samples, dW, dbias and the atomically scattered feature gradient, and the float64 evaluation
# above computes it.  check_exact() asserts those preconditions on a generated case.
TF32_EXACT = 2048
FP32_EXACT = 2.0 ** 24
FP64_EXACT = 2.0 ** 53


def integer_case(B, N, npoint, ns, c_feat, widths, seed=0, bn=False, group_all=False):
    """integer-valued inputs of one scale, on the CPU: dict(xyz (B, N, 3), centres (B, P, 3), feats (B, c_feat, N) or
    None, idx (B, P, ns) int32 (float32 tensors otherwise), layers (layer_params form, float64), grad_out (B, C_last, P)).
    - coordinates on an integer grid and centres that are points of the cloud (GroupAll: the origin and idx = arange(N),
      npoint = 1, ns = N), so xyz[idx] - centre is exact; features in [-3, 3];
    - weights in {-1, 0, 1}: each output row has max(4, ceil(c_in / c_out)) nonzeros (at most c_in) at consecutive
      columns modulo c_in, so every input column is read, the last K chunk and K tail included; biases in {-1, .., 2};
    - idx: random points with a random number of hits per group, padded with the first hit as the ball query pads;
      point N - 1 in the last group of the last scene;
    - grad_out: one nonzero (+-1 or +-2) per group, in channel (group index) mod C_last, so every row tile, statistics
      part and weight-gradient chunk carries gradient;
    - bn: layers with BatchNorm (gamma, beta, running statistics drawn as floats) instead of a bias."""
    g = torch.Generator().manual_seed(seed)
    xyz = torch.randint(0, 8, (B, N, 3), generator=g).float()
    feats = torch.randint(-3, 4, (B, c_feat, N), generator=g).float() if c_feat else None
    if group_all:
        assert npoint == 1 and ns == N
        centres = torch.zeros(B, 1, 3)
        idx = torch.arange(N, dtype=torch.int32).view(1, 1, N).expand(B, 1, N).contiguous()
    else:
        cidx = torch.randint(0, N, (B, npoint), generator=g)
        centres = torch.gather(xyz, 1, cidx[..., None].expand(B, npoint, 3)).contiguous()
        idx = torch.randint(0, N, (B, npoint, ns), generator=g)
        idx[:, :, 0] = cidx                                   # the centre is its own first hit
        idx[-1, -1, min(1, ns - 1)] = N - 1
        hits = torch.randint(1, ns + 1, (B, npoint, 1), generator=g)
        hits[-1, -1] = ns
        idx = torch.where(torch.arange(ns) >= hits, idx[:, :, :1], idx).int().contiguous()
    layers, c_in = [], 3 + c_feat
    for c_out in widths:
        d = min(c_in, max(4, -(-c_in // c_out)))
        w = torch.zeros(c_out, c_in, dtype=torch.float64)
        rows = torch.arange(c_out).repeat_interleave(d)
        cols = (rows * d + torch.arange(d).repeat(c_out)) % c_in
        w[rows, cols] = torch.randint(0, 2, (c_out * d,), generator=g).double() * 2 - 1
        layer = dict(w=w, b=None)
        if bn:
            layer.update(gamma=torch.rand(c_out, generator=g).double() + 0.5, beta=torch.rand(c_out, generator=g).double() - 0.5,
                         rm=torch.randn(c_out, generator=g).double(), rv=torch.rand(c_out, generator=g).double() + 0.5,
                         nbt=3, eps=1e-5, momentum=0.1)
        else:
            layer["b"] = torch.randint(-1, 3, (c_out,), generator=g).double()
        layers.append(layer)
        c_in = c_out
    G, C = B * npoint, widths[-1]
    grp = torch.arange(G)
    gout = torch.zeros(G, C)
    gout[grp, grp % C] = (torch.randint(1, 3, (G,), generator=g) * (torch.randint(0, 2, (G,), generator=g) * 2 - 1)).float()
    grad_out = gout.view(B, npoint, C).transpose(1, 2).contiguous()
    return dict(xyz=xyz, centres=centres, feats=feats, idx=idx, layers=layers, grad_out=grad_out)


def _require(cond, what):
    if not bool(cond):
        raise AssertionError("not an exact case: " + what)


def _integer_within(t, bound, what):
    _require(torch.equal(t, t.round()), what + " is not integer-valued")
    _require(t.abs().max() <= bound if t.numel() else True, "%s reaches %g (bound %g)" % (what, float(t.abs().max()), bound))


def check_exact(case, ref, layers_exact=None, grad_feats_prefill=None):
    """assert that the device path is exact on `case` (integer_case's form) given `ref`, the scale() evaluation of it with
    grad_out (its own decisions: masks and chosen samples that tie to the device's give the same operands):
    - every TF32 operand is an integer of at most TF32_EXACT: layer-0 rows, inner activations, W, and dZ;
    - for every GEMM the same product on absolute values stays below FP32_EXACT, which bounds every partial sum in any
      order: |A| |W|^T (+ |bias|), |dZ|^T |A|, |dZ| |W|, and the feature scatter (with |grad_feats_prefill|), the bias
      gradient sum |dZ|;
    - BN layers: the column sums of z and z^2 stay below FP64_EXACT.
    layers_exact: how many leading layers to check (default all; a BN chain is exact in layer 0 only, and without its
    backward).  Returns the bound of the feature scatter, (B, c_feat, N) (None without it), for callers that add
    several scales into one feature gradient."""
    layers = case["layers"]
    dev = ref["out"].device
    L = len(layers) if layers_exact is None else layers_exact
    a = rows0(case["xyz"], case["centres"], case["feats"], case["idx"], dev)
    backward = "dz" in ref and all("gamma" not in d for d in layers)
    scatter = None
    for l in range(L):
        d = layers[l]
        w = d["w"].to(dev)
        _integer_within(a, TF32_EXACT, "layer %d input" % l)
        _integer_within(w, TF32_EXACT, "layer %d weight" % l)
        fwd = a.abs() @ w.abs().t()
        if d["b"] is not None:
            fwd += d["b"].to(dev).abs()
        _require(fwd.max() < FP32_EXACT, "layer %d forward |A| |W|^T reaches %g" % (l, float(fwd.max())))
        del fwd
        if "gamma" in d:
            z = a @ w.t()
            _require(z.abs().sum(0).max() < FP64_EXACT and (z * z).sum(0).max() < FP64_EXACT,
                     "layer %d BN column sums reach 2^53" % l)
            del z
        if backward:
            dz = ref["dz"][l]
            _integer_within(dz, TF32_EXACT, "layer %d dZ" % l)
            dw = dz.abs().t() @ a.abs()
            _require(dw.max() < FP32_EXACT, "layer %d weight gradient |dZ|^T |A| reaches %g" % (l, float(dw.max())))
            _require(dz.abs().sum(0).max() < FP32_EXACT, "layer %d bias gradient reaches 2^24" % l)
            da = dz.abs() @ w.abs()
            _require(da.max() < FP32_EXACT, "layer %d dA |dZ| |W| reaches %g" % (l, float(da.max())))
            if l == 0 and case["feats"] is not None:
                B, c_feat, N = case["feats"].shape
                idx = case["idx"].long().to(dev)
                point = (idx + torch.arange(B, device=dev)[:, None, None] * N).reshape(-1)
                acc = torch.zeros(B * N, c_feat, dtype=torch.float64, device=dev).index_add_(0, point, da[:, 3:])
                if grad_feats_prefill is not None:
                    acc += grad_feats_prefill.double().to(dev).transpose(1, 2).reshape(B * N, c_feat).abs()
                _require(acc.max() < FP32_EXACT, "feature gradient scatter reaches %g" % float(acc.max()))
                scatter = acc.view(B, N, c_feat).transpose(1, 2)
            del dw, da
        a = torch.relu(ref["pre"][l])
    return scatter



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
