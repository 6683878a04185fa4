"""A float64 evaluation of what an eval-mode module computes from its own torch parameters, with a per-element bound on
|fused kernel output - evaluation|.

mlp_reference.py checks the chain kernel against the weights read back from the packed image.  This reference starts
one step earlier, at the module: conv weight and bias, BatchNorm (x - running_mean) / sqrt(running_var + eps) * weight +
bias, ReLU (not on the linear last layer of the RPN heads), max-pool over the samples of an SA centre, inverse-distance
interpolation plus skip concat for FP.  So a wrong fold, cache, channel offset, projection split or head block shows up
as elements outside the bound, however small the channel is next to the tensor's largest value.

Everything runs in torch float64 on the device of the inputs.  Index work (FPS centres, ball-query indices, 3-NN
indices and weights) is taken from the device's own outputs; those are pinned exactly elsewhere.

The bound reuses mlp_reference's model -- gamma(K) for a K_pad-term fp32 accumulation, U32 for one fp32 rounding,
TF32_HALF_ULP for one round-to-nearest to TF32, ReLU and max 1-Lipschitz (max-pooled bounds for the SA max) -- and adds
the terms that lie between the module and the packed image:

  inverse std   fl(gamma / fl(sqrt(fl(var + fl(eps))))): INV_REL = 4 U32 relative (eps rounded, add, sqrt, divide)
  weight        BN layers: W * inv rounded to fp32 (fold_scale) or the scale inv_f kept apart (fold_scale=False), then the
                packer's rna to TF32: RHO_BN = (1 + 5 U32)(1 + 2^-11) - 1 relative to |inv W|.  Layers without BN:
                the rna alone, 2^-11 |W|.  Identity columns ([I | W0s] of a projected FP level) are exact.
  shift         beta - fl(mean * inv_f) (+ fl(inv_f * b)), each product and sum rounded once:
                SHIFT_REL = 8 U32 of |beta| + |mean * inv| + |inv * b|; a BN-free layer's shift is its bias, exact
  epilogue      one fp32 rounding of s z + t (fmaf; s = 1 when the scale is folded), U32 (|y| + bound)
  activations   rounded to TF32 between the layers of a chain, 2^-11 (|y| + bound)
  SA layer 0    fl(x - centre) then tf32_rn: ((1 + U32)(1 + 2^-11) - 1) |x - centre|; features tf32_rn: 2^-11 |f|
  FP layer 0    interpolation fma(w2,p2, fma(w0,p0, w1*p1)): FP_INTERP_ROUNDINGS of sum |w_k p_k|, then tf32_rn;
                skip channels tf32_rn
  projected FP  the projection known @ (inv W0k)^T is a linear row chain: its accumulation over round_up(c_known, 32)
                terms of tf32_rn(known), the weight rounding and its fp32 store; the projected rows are interpolated
                (the interpolation roundings, over |w_k| (|P_k| + bound_k)) and rounded to TF32; then layer 0 runs over
                [I | inv W0s] with the original shift
  rows          tf32_rn of every input column, 2^-11 |x|

A layer with input a (bound e), folded weight Wt = inv W, weight error Wr = rho |Wt| and M = |Wt| + Wr:
    bound = gamma(K_pad) (|a| + e) M^T + e M^T + |a| Wr^T + shift bound, then the epilogue and TF32 roundings above.
"""
import gc

import torch

import mlp_reference as R
from pointrcnn_b200 import mlp_chain

U32, HALF = R.U32, R.TF32_HALF_ULP
INV_REL = 4 * U32
RHO_BN = (1 + 5 * U32) * (1 + HALF) - 1
SHIFT_REL = 8 * U32
SUB_REL = (1 + U32) * (1 + HALF) - 1


class Layer:
    """one conv [+ BN] block in float64: Wt = inv W (c_out, c_in), rho its relative weight error, shift T and its bound"""

    def __init__(self, conv, bn, relu, device):
        co = conv.out_channels
        f64 = dict(dtype=torch.float64, device=device)
        W = conv.weight.detach().to(**f64).reshape(co, -1)
        b = conv.bias.detach().to(**f64) if conv.bias is not None else torch.zeros(co, **f64)
        self.relu = relu
        if bn is None:
            self.Wt, self.rho, self.shift, self.eshift = W, HALF, b, torch.zeros(co, **f64)
            return
        inv = bn.weight.detach().to(**f64) / torch.sqrt(bn.running_var.detach().to(**f64) + bn.eps)
        mean, beta = bn.running_mean.detach().to(**f64), bn.bias.detach().to(**f64)
        self.Wt, self.rho = inv[:, None] * W, RHO_BN
        self.shift = beta - mean * inv + inv * b
        self.eshift = SHIFT_REL * (beta.abs() + (mean * inv).abs() + (inv * b).abs())


def layers_of(blocks, device):
    """[Layer] of pointnet2_modules.read_block triples"""
    return [Layer(conv, bn, relu, device) for conv, bn, relu in blocks]


def mlp_layers(mlp, device):
    from pointrcnn_b200.pointnet2 import pointnet2_modules as pm
    blocks = pm.read_mlp(mlp)
    assert blocks is not None, "not a SharedMLP the fused path runs"
    return layers_of(blocks, device)


def apply(a, e, Wt, Wr, k_pad, shift, eshift, relu, rounded):
    """one layer: (y, bound).  Wr: the absolute weight error per element (same shape as Wt)"""
    Wa = Wt.abs()
    M = Wa + Wr
    aa = a.abs()
    z = a @ Wt.T
    ez = R.gamma(k_pad) * ((aa + e) @ M.T) + e @ M.T + aa @ Wr.T
    y = z + shift
    ey = ez + eshift
    ey = ey + U32 * (y.abs() + ey)                 # the epilogue's fmaf
    if relu:
        y = y.clamp_min(0)
    if rounded:
        ey = ey + HALF * (y.abs() + ey)            # activation rounded to TF32 for the next layer
    return y, ey


def chain(layers, a, e, k_pad0, k_pads=None):
    """run `layers` over rows a (bound e); layer 0 contracts over k_pad0 packed columns, layer l over k_pads[l] (default:
    its input width rounded up to 32).  The last layer's output is not rounded to TF32."""
    for l, ly in enumerate(layers):
        last = l == len(layers) - 1
        k = k_pad0 if l == 0 else (k_pads[l] if k_pads else R.round_up(ly.Wt.shape[1], 32))
        a, e = apply(a, e, ly.Wt, ly.rho * ly.Wt.abs(), k, ly.shift, ly.eshift, ly.relu, not last)
    return a, e


def k_pad0(kind, split, c_in):
    return len(R.k_order(kind, split, c_in)[0])


# ------------------------------------------------------------------------------------------------ modules
def sa_scale(mlp, xyz, feats, centres, idx):
    """one scale of an SA module: xyz (B,N,3), feats (B,C,N) or None, centres (B,npoint,3) (zeros for GroupAll), idx
    (B,npoint,ns) -> (y, bound) (B, c_last, npoint), max-pooled over the ns samples.  One scene at a time."""
    dev = xyz.device
    layers = mlp_layers(mlp, dev)
    c_feat = 0 if feats is None else feats.size(1)
    k0 = k_pad0(mlp_chain.SA, c_feat, 3 + c_feat)
    ys, es = [], []
    for b in range(xyz.size(0)):
        npoint, ns = idx.shape[1:]
        i = idx[b].long().reshape(-1)
        rel = xyz[b].double()[i].view(npoint, ns, 3) - centres[b].double()[:, None, :]
        a, e = [rel], [SUB_REL * rel.abs()]
        if c_feat:
            f = feats[b].double().T[i].view(npoint, ns, c_feat)
            a.append(f)
            e.append(HALF * f.abs())
        a, e = torch.cat(a, -1).view(npoint * ns, -1), torch.cat(e, -1).view(npoint * ns, -1)
        y, ey = chain(layers, a, e, k0)
        ys.append(y.view(npoint, ns, -1).amax(1).T)
        es.append(ey.view(npoint, ns, -1).amax(1).T)
    return torch.stack(ys), torch.stack(es)


def _interp(p, ep, idx, w):
    """inverse-distance interpolation of rows p (m, c) (bound ep) at idx / w (n, 3), rounded to TF32 as the kernel gathers"""
    i, w = idx.long(), w.double()
    terms = [w[:, k:k + 1] * p[i[:, k]] for k in range(3)]
    v = terms[0] + terms[1] + terms[2]
    mag = sum(w[:, k:k + 1].abs() * (p[i[:, k]].abs() + ep[i[:, k]]) for k in range(3))
    ev = sum(w[:, k:k + 1].abs() * ep[i[:, k]] for k in range(3)) + R.FP_INTERP_ROUNDINGS * mag
    return v, ev + HALF * (v.abs() + ev)


def fp_module(mlp, idx, weight, skip, known_feats, projected):
    """an FP module: idx / weight (B,n,3) from the 3-NN, skip (B,c_skip,n) or None, known_feats (B,c_known,m) ->
    (y, bound) (B, c_last, n).  projected: layer 0 split into a per-known-point projection and [I | W0s] (what
    PointnetFPModule.fused_mlp runs when it projects)."""
    dev = known_feats.device
    layers = mlp_layers(mlp, dev)
    c_known = known_feats.size(1)
    c_skip = 0 if skip is None else skip.size(1)
    L0 = layers[0]
    c1 = L0.Wt.shape[0]
    ys, es = [], []
    for b in range(idx.size(0)):
        known = known_feats[b].double().T
        if projected:
            Wk = L0.Wt[:, :c_known]
            zero = torch.zeros(c1, dtype=torch.float64, device=dev)
            P, eP = apply(known, HALF * known.abs(), Wk, L0.rho * Wk.abs(), R.round_up(c_known, 32), zero, zero, False, False)
            v, ev = _interp(P, eP, idx[b], weight[b])
            Wt0 = torch.cat([torch.eye(c1, dtype=torch.float64, device=dev), L0.Wt[:, c_known:]], 1)
            Wr0 = torch.cat([torch.zeros(c1, c1, dtype=torch.float64, device=dev), L0.rho * L0.Wt[:, c_known:].abs()], 1)
            k0 = k_pad0(mlp_chain.FP, c1, c1 + c_skip)
        else:
            v, ev = _interp(known, torch.zeros_like(known), idx[b], weight[b])
            Wt0, Wr0 = L0.Wt, L0.rho * L0.Wt.abs()
            k0 = k_pad0(mlp_chain.FP, c_known, c_known + c_skip)
        a, e = [v], [ev]
        if c_skip:
            s = skip[b].double().T
            a.append(s)
            e.append(HALF * s.abs())
        a, e = torch.cat(a, 1), torch.cat(e, 1)
        y, ey = apply(a, e, Wt0, Wr0, k0, L0.shift, L0.eshift, True, len(layers) > 1)
        y, ey = chain(layers[1:], y, ey, R.round_up(c1, 32)) if len(layers) > 1 else (y, ey)
        ys.append(y.T)
        es.append(ey.T)
    return torch.stack(ys), torch.stack(es)


def rows_mlp(mlp, a, b=None):
    """pointnet2_modules.rows_mlp: the SharedMLP over rows [a | b] -> (y, bound) (rows, c_last)"""
    x = a.double() if b is None else torch.cat([a.double(), b.double()], 1)
    kind, split = mlp_chain.rows_layout(a.size(1), 0 if b is None else b.size(1))
    return chain(mlp_layers(mlp, a.device), x, HALF * x.abs(), k_pad0(kind, split, x.size(1)))


def heads(cls_seq, reg_seq, rows):
    """the eval-mode RPN heads over point rows (rows, C): [(y, bound) of cls, (y, bound) of reg].  Each stack is
    evaluated on its own; the fused chain's second layer contracts over both hidden layers (its K_pad)."""
    from pointrcnn_b200.rpn import heads as H
    stacks = [layers_of(H._layers(seq), rows.device) for seq in (cls_seq, reg_seq)]
    k1 = R.round_up(sum(s[0].Wt.shape[0] for s in stacks), 32)
    x = rows.double()
    return [chain(s, x, HALF * x.abs(), R.round_up(x.size(1), 32), k_pads=[None, k1]) for s in stacks]


# ------------------------------------------------------------------------------------------------ test modules
def seeded(module, seed):
    """random conv weights and biases; BN with gammas of both signs and non-zero means.  Every seventh channel is nearly
    dead: running_var 1e-4, where eps moves the inverse std by 5%, and a gamma 20x smaller, so the channel is no larger
    than the others.  Channels 3, 14, 25, ... are small: a gamma 100x smaller, so their values sit far below the largest
    value of the output."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for m in module.modules():
            if isinstance(m, (torch.nn.Conv1d, torch.nn.Conv2d)):
                m.weight.copy_(torch.randn(m.weight.shape, generator=g) * (2.0 / m.weight[0].numel()) ** 0.5)
                if m.bias is not None:
                    m.bias.copy_(torch.randn(m.bias.shape, generator=g) * 0.1)
            elif isinstance(m, (torch.nn.BatchNorm1d, torch.nn.BatchNorm2d)):
                c = m.num_features
                sign = torch.where(torch.rand(c, generator=g) < 0.3, -1.0, 1.0)
                m.weight.copy_((torch.rand(c, generator=g) + 0.5) * sign)
                m.bias.copy_(torch.randn(c, generator=g) * 0.1)
                m.running_mean.copy_(torch.randn(c, generator=g) * 0.2)
                var = torch.rand(c, generator=g) + 0.5
                var[::7] = 1e-4
                m.weight[::7] *= 0.05
                m.weight[3::11] *= 0.01
                m.running_var.copy_(var)
    return module.eval()


def replace_parameter(module, name, data):
    """module.<name> replaced by nn.Parameter(data), with `data` allocated by the caller while the old parameter is still
    alive: the new Parameter object then takes the slot the old one frees, so when nothing else holds the old parameter
    the new one has its id() (and, like it if it was fresh, version 0).  Returns whether the id() was reused.  The cyclic
    collector is held off meanwhile: a collection between the two steps frees other objects whose slots come first."""
    old_id = id(getattr(module, name))
    enabled = gc.isenabled()
    gc.disable()
    try:
        delattr(module, name)
        setattr(module, name, torch.nn.Parameter(data))
    finally:
        if enabled:
            gc.enable()
    return id(getattr(module, name)) == old_id


# ------------------------------------------------------------------------------------------------ the check
def check(got, ref, bound):
    """(every element inside its bound, max err / bound, number outside); NaN or Inf in `got` is outside"""
    err = (got.double() - ref).abs()
    ok = err <= bound
    ratio = torch.where(err == 0, torch.zeros_like(err), err / bound)
    ratio = torch.where(torch.isfinite(got), ratio, torch.full_like(err, float("inf")))
    return bool(ok.all()), float(ratio.max()) if ratio.numel() else 0.0, int((~ok).sum())


def old_tol_passes(got, ref, tol=2e-3):
    """the norm-wise check this reference replaces: max |err| <= tol * max |ref|"""
    return float((got.double() - ref).abs().max()) <= tol * float(ref.abs().max())
