"""Float64 CPU reference of one PointnetFPModule in training mode: three-tap interpolation, skip concatenation, 1-3 layers
of 1x1 conv + [batch-statistics BatchNorm | conv bias] + ReLU, and the backward of all of it, written out explicitly.

Layer 0 runs in either order: "plain" (interpolate, then W0) or "projected" (project the known points through the
interpolated columns Wi, then interpolate; the backward through G = I^T dZ0).  In exact arithmetic both are the same.
`mutant` plants one mistake, so the tests can show the tolerances of `compare` catch it.
"""
import numpy as np
import torch

MUTANTS = ("no_bn_term", "unbiased", "no_relu_mask", "wrong_tap", "swap_cols")


def _interp(x, idx, w, mutant=None):
    """x (B, m, C) point-major, idx / w (B, n, 3) -> (B, n, C) = sum_t w_t x[idx_t]"""
    B, n, _ = idx.shape
    taps = idx.long()
    if mutant == "wrong_tap":
        taps = taps[..., [1, 0, 2]]
    g = torch.stack([x[b][taps[b]] for b in range(B)])          # (B, n, 3, C)
    return (g * w.unsqueeze(-1)).sum(2)


def _interp_t(d, idx, w, m):
    """the transpose: d (B, n, C) -> (B, m, C) = I^T d"""
    B, n, C = d.shape
    out = torch.zeros((B, m, C), dtype=d.dtype)
    for b in range(B):
        for t in range(3):
            out[b].index_add_(0, idx[b, :, t].long(), d[b] * w[b, :, t:t + 1])
    return out


def forward(known, skip, idx, w, layers, bn, eps=1e-5, order="plain", mutant=None):
    """known (B, ci, m), skip (B, cs, n) or None, idx / w (B, n, 3); layers: list of dict(W (co, ci), bias, gamma, beta).
    -> (out (B, C_last, n), cache)"""
    known, w = known.double(), w.double()
    skip = skip.double() if skip is not None else None
    B, ci, m = known.shape
    n = idx.shape[1]
    F = known.transpose(1, 2)                                   # (B, m, ci)
    S = skip.transpose(1, 2) if skip is not None else torch.zeros((B, n, 0), dtype=torch.float64)
    W0 = layers[0]["W"].double()
    Wi, Ws = W0[:, :ci], W0[:, ci:]
    if mutant == "swap_cols":
        Wi, Ws = W0[:, W0.shape[1] - ci:], W0[:, :W0.shape[1] - ci]
    if order == "plain":
        Z = _interp(F, idx, w, mutant) @ Wi.T + S @ Ws.T
    else:
        Z = _interp(F @ Wi.T, idx, w, mutant) + S @ Ws.T
    cache = dict(F=F, S=S, idx=idx, w=w, m=m, ci=ci, layers=layers, bn=bn, order=order, mutant=mutant, zs=[], xs=[], ys=[], st=[])
    rows = B * n
    for l, L in enumerate(layers):
        if l:
            Z = cache["ys"][-1] @ L["W"].double().T
        Zr = Z.reshape(rows, -1)
        if bn:
            mean = Zr.mean(0)
            var = Zr.var(0, unbiased=(mutant == "unbiased"))
            invstd = 1.0 / torch.sqrt(var + eps)
            xhat = (Zr - mean) * invstd
            pre = xhat * L["gamma"].double() + L["beta"].double()
            cache["st"].append((mean, Zr.var(0, unbiased=True), invstd))
        else:
            xhat = Zr
            pre = Zr + (L["bias"].double() if L.get("bias") is not None else 0.0)
        y = torch.relu(pre)
        cache["zs"].append(Zr)
        cache["xs"].append((xhat, pre))
        cache["ys"].append(y.reshape(B, n, -1))
    out = cache["ys"][-1].transpose(1, 2).contiguous()
    return out, cache


def backward(cache, gout, masks=None):
    """gout (B, C_last, n) -> dict(W=[..], bias=[..], gamma=[..], beta=[..], known (B, ci, m), skip (B, cs, n)).
    masks: per layer the (rows, C) ReLU decisions to use instead of the reference's own (a device's, so that values
    within rounding of zero do not flip a whole row's gradient)"""
    layers, bn, mutant = cache["layers"], cache["bn"], cache["mutant"]
    B, n, _ = cache["ys"][-1].shape
    rows = B * n
    g = gout.double().transpose(1, 2).reshape(rows, -1)
    res = dict(W=[None] * len(layers), bias=[None] * len(layers), gamma=[None] * len(layers), beta=[None] * len(layers))
    for l in range(len(layers) - 1, -1, -1):
        xhat, pre = cache["xs"][l]
        if mutant != "no_relu_mask":
            g = g * (masks[l].cpu() if masks is not None else (pre > 0))
        if bn:
            gam = layers[l]["gamma"].double()
            invstd = cache["st"][l][2]
            res["gamma"][l] = (g * xhat).sum(0)
            res["beta"][l] = g.sum(0)
            if mutant == "no_bn_term":
                dz = gam * invstd * (g - g.mean(0))
            else:
                dz = gam * invstd * (g - g.mean(0) - xhat * (g * xhat).mean(0))
        else:
            res["bias"][l] = g.sum(0)
            dz = g
        if l:
            a = cache["ys"][l - 1].reshape(rows, -1)
            res["W"][l] = dz.T @ a
            g = dz @ layers[l]["W"].double()
            continue
        ci, m = cache["ci"], cache["m"]
        F, S, idx, w = cache["F"], cache["S"], cache["idx"], cache["w"]
        W0 = layers[0]["W"].double()
        d3 = dz.reshape(B, n, -1)
        if cache["order"] == "plain":
            X = torch.cat([_interp(F, idx, w, mutant), S], 2).reshape(rows, -1)
            res["W"][0] = dz.T @ X
            dX = (dz @ W0).reshape(B, n, -1)
            res["known"] = _interp_t(dX[..., :ci], idx, w, m).transpose(1, 2)
            res["skip"] = dX[..., ci:].transpose(1, 2)
        else:
            G = _interp_t(d3, idx, w, m)                         # (B, m, c1)
            Gr = G.reshape(B * m, -1)
            dWi = Gr.T @ F.reshape(B * m, -1)
            dWs = dz.T @ S.reshape(rows, -1)
            res["W"][0] = torch.cat([dWi, dWs], 1)
            res["known"] = (G @ W0[:, :ci]).transpose(1, 2)
            res["skip"] = (d3 @ W0[:, ci:]).transpose(1, 2)
    return res


def compare(ref, got, kind):
    """(ok, message): forward within 2e-3 max|ref|; gradients within 5e-3 max|ref| elementwise and 2e-3 relative Frobenius"""
    ref, got = ref.double(), got.double().cpu()
    scale = max(float(ref.abs().max()), 1e-30)
    err = float((ref - got).abs().max())
    if kind == "fwd":
        return err <= 2e-3 * scale, "max err %.3g vs %.3g" % (err, 2e-3 * scale)
    fro = float(torch.linalg.norm(ref - got) / max(float(torch.linalg.norm(ref)), 1e-30))
    return err <= 5e-3 * scale and fro <= 2e-3, "max err %.3g vs %.3g, rel fro %.3g" % (err, 5e-3 * scale, fro)


# ------------------------------------------------------------------------------------------------ integer cases
def integer_case(B, n, m, ci, cs, widths, seed=0, taps="half"):
    """an FP case whose device result has one right answer: integer features in [-3, 3], biases in {-1..2}, sparse weights
    in {-1, 0, 1} that read every input column, and interpolation weights exact in fp32 ("half": 1/2, 1/4, 1/4 on three
    distinct known points; "onehot": 1, 0, 0).  Bias chains only (batch statistics are not exact).
    -> dict(known, skip, idx, w, layers, gout)"""
    g = np.random.default_rng(seed)
    known = torch.from_numpy(g.integers(-3, 4, (B, ci, m)).astype(np.float32))
    skip = torch.from_numpy(g.integers(-3, 4, (B, cs, n)).astype(np.float32)) if cs else None
    idx = np.stack([np.stack([g.choice(m, 3, replace=m < 3) for _ in range(n)]) for _ in range(B)]).astype(np.int32)
    idx[:, -1, 0] = m - 1
    wt = [0.5, 0.25, 0.25] if taps == "half" else [1.0, 0.0, 0.0]
    w = torch.tensor(wt, dtype=torch.float32).expand(B, n, 3).contiguous()
    layers, c_in = [], ci + cs
    for co in widths:
        W = g.choice([-1.0, 0.0, 0.0, 1.0], (co, c_in)).astype(np.float32)
        W[np.arange(c_in) % co, np.arange(c_in)] = 1.0             # every input column is read
        layers.append(dict(W=torch.from_numpy(W), bias=torch.from_numpy(g.integers(-1, 3, co).astype(np.float32))))
        c_in = co
    gout = torch.from_numpy(g.integers(-1, 2, (B, widths[-1], n)).astype(np.float32))
    return dict(known=known, skip=skip, idx=torch.from_numpy(idx), w=w, layers=layers, gout=gout)


def _tf32_exact(t):
    """every element is a float32 whose low 13 mantissa bits are zero (TF32 keeps it as it is)"""
    f = t.double().numpy().astype(np.float32)
    return np.array_equal(f.astype(np.float64), t.double().numpy()) and not np.any(f.view(np.uint32) & 0x1FFF)


def check_exact(case, cache, out, grads):
    """asserts the preconditions of a bit-exact comparison: every GEMM operand the device stages (interpolated features,
    skip, weights, inner activations, dZ, G) is exact in TF32, and every value and partial sum is a multiple of 1/4 below
    2^22, so fp32 arithmetic in any order gives the float64 answer; cache / out / grads: the float64 reference's"""
    lim = 2.0 ** 22
    ops = [_interp(cache["F"], cache["idx"], cache["w"]), cache["S"]] + [L["W"] for L in case["layers"]]
    ops += [y for y in cache["ys"][:-1]]
    B, n, _ = cache["ys"][-1].shape
    g = case["gout"].double().transpose(1, 2).reshape(B * n, -1)
    for l in range(len(case["layers"]) - 1, -1, -1):
        g = g * (cache["xs"][l][1] > 0)
        ops.append(g)
        if l == 0:
            ops.append(_interp_t(g.reshape(B, n, -1), cache["idx"], cache["w"], cache["m"]))
        else:
            g = g @ case["layers"][l]["W"].double()
    for t in ops:
        assert _tf32_exact(t), "a GEMM operand is not exact in TF32"
    vals = [out, grads["known"]] + [t for k in ("W", "bias") for t in grads[k] if t is not None]
    vals += [grads["skip"]] if grads.get("skip") is not None else []
    vals += [z.abs().sum(1) for z in cache["zs"]]
    for t in vals:
        t = t.double()
        assert float(t.abs().max()) < lim, "a value of %g reaches 2^22" % float(t.abs().max())
        assert torch.equal(t * 4, torch.round(t * 4)), "a value is not a multiple of 1/4"
