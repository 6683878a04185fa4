"""A float64 reference of the SA and FP training kernels (csrc/sa_train.cu) with a per-element error bound on every
quantity they produce: the pooled / propagated outputs, the running statistics, and every gradient.

Every float64 quantity x carries a companion e(x) >= |device - x|, computed by the same float64 operations on absolute
values (sum |a| |w| for each GEMM).  The reference replays the device stage by stage: each layer is evaluated in float64
from the device's own saved output of the stage before (its Z and fp32 statistics), and that output is checked in turn
(every Z element, every statistic).  A worst-case bound carried through a BatchNorm grows with the ratio of sum |w| |a|
to the batch spread, several fold per layer, so an end-to-end bound over three BN layers says nothing; chained stage by
stage the bounds stay within a few TF32 roundings and still pin every stage.  The decisions are the device's: the ReLU
masks are the sign of fma(a, z, b) of its saved Z and statistics (exact in float64), the chosen samples its own; they are
checked against the reference (`relu_flips`, `pool_choices`).

The terms, with u = 2^-24 (fp32 round to nearest), t = 2^-11 (cvt.rn.tf32, half an ulp of 10 stored bits) and
u64 = 2^-53:
  TF32 operand     every GEMM operand x +- e is rounded to TF32 as it is staged: e + t (|x| + e)          (tf32_in)
  GEMM             mma.sync m16n8k8 TF32 products are exact in fp32; the fp32 accumulation over K terms loses at most
                   gamma(K) = (K8 + 2) 2^-22 of sum |x~| |y~| (K8: K rounded up to 8; two ulps per added term, as
                   tests/mlp_reference.py assumes for wgmma).  Bound (1 + gamma) (|X| + eX)(|Y| + eY) - |X| |Y|  (gemm)
                   K is the reduction length of one fp32 accumulator: c_in (forward), c_out (dA), the row chunk of the
                   weight-gradient split (dW, st_wsplit), c_known for the projection P = F Wi^T, c_skip for S Ws^T
  dW partials      the row-chunk partials summed in float64 (g64(parts) of their magnitude), stored as fp32 (u)
  float64 sums     column sums of z, z^2, g, g xhat: n u64 of the summed magnitude, any order               (g64)
  BN statistics    of the device's Z: mean g64 (n + 1) of mean |z|; variance 3 g64(n + 4) mean(z^2) (E[z^2] - mean^2 in
                   float64, the term that grows with |mean| / std); invstd by the mean value theorem on (var + eps)^-1/2;
                   mean, invstd, a = gamma invstd, b = beta - mean a stored as fp32 (u)
  pre-activation   fma(a32, z, b32) against gamma xhat + beta (the ReLU decision check): u |a| |z| (a32) + u |b| (b32) +
                   |gamma| e_invstd |z - mean| + |a| e_mean + u |p| -- with |mean| >> std, u |a| (|z| + |mean|)
  activations      relu(fma(a32, z, b32)) of the device's Z and statistics: one fp32 rounding (u)
  xhat             fl(fl(z - mean32) invstd32): (e_mean32 + u |z - mean|) invstd + |z - mean| e_invstd32 + u |xhat|
  BN backward      sums sum(g), sum(g xhat) (e_g, e_xhat, g64), stored as fp32 (dbeta, dgamma) and as the fp32 means
                   mg0, mg1; dZ = a32 (g - mg0 - xhat mg1) in fp32: three roundings of |g| + |mg0| + |xhat mg1| inside the
                   bracket, one of the product, and the error of a32
  feature scatter  fp32 adds per point, atomic (any order) or ordered (per scale in list order, then scale by scale):
                   both are cnt - 1 roundings of at most the point's sum of |v| (cnt: the rows that reference the point,
                   over all scales)                                                                              (gsum)
  FP interpolation fma(w2, P2, fma(w0, P0, w1 P1)) over the fp32 projection P: 3 roundings of sum w |P|, then the add to
                   S Ws^T (u); the transpose G = I^T dZ0 is an fma chain per known point: cnt roundings
The check is |device - reference| <= bound for every element (`ratio` is the largest error / bound).  The module is
device-agnostic: the GPU tests evaluate it on the GPU.
"""
import math

import torch

from mlp_reference import tf32_rn

U = 2.0 ** -24
T = 2.0 ** -11
U64 = 2.0 ** -53
ROW_TILE, BK, WCTAS = 128, 32, 528


def gamma(k):
    return (-(-int(k) // 8) * 8 + 2) * 2.0 ** -22


def g64(n):
    return n * U64


def gsum(cnt):
    """relative error of an fp32 sum of cnt terms in any order (elementwise over a count tensor)"""
    k = (cnt.double() - 1).clamp_min(0)
    return k * U / (1 - k * U)


def wsplit(rows, cout, cin):
    """(chunk, parts) of a weight-gradient GEMM's row split, as st_wsplit computes them"""
    tiles = -(-cout // 64) * -(-cin // 64)
    parts = max(min(-(-WCTAS // tiles), -(-rows // 256)), 1)
    chunk = -(-(-(-rows // parts)) // BK) * BK
    return chunk, -(-rows // chunk)


def tf32_in(x, e):
    return e + T * (x.abs() + e)


def gemm(X, eX, Y, eY, K):
    """X @ Y as the device computes it from operands within eX / eY of X / Y -> (value, bound, magnitude)"""
    eX, eY = tf32_in(X, eX), tf32_in(Y, eY)
    ax, ay = X.abs(), Y.abs()
    M = (ax + eX) @ (ay + eY)
    return X @ Y, (1 + gamma(K)) * M - ax @ ay, (1 + gamma(K)) * M


def weight_grad(dz, e_dz, a, e_a, K, parts, store=True):
    """dW = dZ^T A through the row-chunk partials, their float64 sum and (store) the fp32 store"""
    v, e, M = gemm(dz.t(), e_dz.t(), a, e_a, K)
    e = e + g64(parts) * M
    return v, _store32(v, e) if store else e


def _store32(v, e):
    """a float64 value stored as fp32"""
    return e + U * (v.abs() + e)


# ------------------------------------------------------------------------------------------------ the layer stack
def device_act(z, st):
    """relu(fma(a, z, b)) of the device's saved Z and fp32 statistics (4, C), in float64 (before its fp32 rounding)"""
    return (st[2].double() * z.double() + st[3].double()).clamp_min(0)


class Stack:
    """the layers of one SA scale or FP module replayed stage by stage from the device's saved Z and statistics.
    layers: sa_train_reference.layer_params form; zs: the device's Z per layer (rows, C_l); stats: its (4, C_l) rows (mean,
    invstd, a, b) per layer.  Every check lands in self.checks as (device value, reference, bound).
    A bias chain (no BN) has no sum across rows but its parameter gradients, so it may be replayed a part of the rows at a
    time: rows_total is then the device's row count (it sets the weight-gradient split and the float64 sum lengths) and
    store=False leaves the parameter gradients without their final fp32 rounding, for the caller to add the parts and
    apply it once (finish_grads)."""

    def __init__(self, layers, zs, stats, dev, rows_total=None, store=True):
        self.rows_total, self.store = rows_total, store
        self.layers = [{k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in d.items()} for d in layers]
        self.bn = "gamma" in layers[0]
        assert rows_total is None or not self.bn, "batch statistics need every row at once"
        self.L = len(layers)
        self.zs = [z.to(dev) for z in zs]                     # fp32: float64 copies of every layer would double the memory
        self.stats = [s.to(dev).double() for s in stats]
        self.checks, self.st, self.flips = {}, [], 0.0     # flips: relu_flips of the device's masks against the reference
        self.masks = [(s[2] * z.double() + s[3]) > 0 for z, s in zip(self.zs, self.stats)]   # exactly the device's ReLU decisions

    def act(self, l):
        """the device's activation of layer l in float64"""
        return device_act(self.zs[l], self.stats[l])

    def check(self, name, got, ref, bound):
        self.checks[name] = (got, ref, bound)

    def forward(self, z0_ref, ez0):
        """checks layer 0's Z against (z0_ref, ez0), then every later Z against the GEMM of the device's activation, and
        every layer's statistics and running statistics against float64 ones of the device's Z"""
        self.check("z0", self.zs[0], z0_ref, ez0)
        for l in range(self.L):
            if l:
                w = self.layers[l]["w"]
                a = self.act(l - 1)
                z, ez, _ = gemm(a, U * a, w.t(), 0, w.shape[1])
                del a
                self.check("z%d" % l, self.zs[l], z, ez)
            self._stats(l)

    def _stats(self, l):
        d, z, dev_st = self.layers[l], self.zs[l].double(), self.stats[l]
        n = z.shape[0]
        s = {}
        if self.bn:
            mean = z.mean(0)
            dz = z - mean
            var = (dz * dz).mean(0)
            em = g64(n + 1) * z.abs().mean(0)
            evar = 3 * g64(n + 4) * (z * z).mean(0)
            eps = d["eps"]
            inv = 1.0 / torch.sqrt(var + eps)
            einv = 0.5 * evar * ((var - evar).clamp_min(0) + eps) ** -1.5 + 4 * U64 * inv
            ga, be = d["gamma"], d["beta"]
            a = ga * inv
            b = be - mean * a
            ea64 = ga.abs() * einv
            eb64 = ga.abs() * (em * inv + (mean.abs() + em) * einv) + 3 * U64 * (mean * a).abs()
            s.update(mean=mean, inv=inv, a=a, ea32=_store32(a, ea64), em32=_store32(mean, em), einv32=_store32(inv, einv))
            for r, (v, e) in enumerate(((mean, em), (inv, einv), (a, ea64), (b, eb64))):
                self.check("%s%d" % (("mean", "invstd", "a", "b")[r], l), dev_st[r], v, _store32(v, e))
            pre = a * dz + be
            epre = U * (a.abs() + ea64) * z.abs() + _store32(b, eb64) + ga.abs() * einv * (dz.abs() + em) + a.abs() * em
            self.flips = max(self.flips, relu_flips([self.masks[l]], [pre], [epre + U * (pre.abs() + epre)]))
            del pre, epre, dz
            m = d["momentum"]
            rm = (1 - m) * d["rm"] + m * mean
            rv = (1 - m) * d["rv"] + m * var * n / (n - 1)
            s["running"] = (rm, _store32(rm, m * em), rv, _store32(rv, m * evar * n / (n - 1)))
        else:
            bias = d["b"] if d["b"] is not None else torch.zeros_like(z[0])
            one, zero = torch.ones_like(bias), torch.zeros_like(bias)
            for r, v in enumerate((zero, one, one, bias)):
                self.check("%s%d" % (("mean", "invstd", "a", "b")[r], l), dev_st[r], v, zero)
            s.update(a=one, ea32=zero, running=None)
            self.flips = max(self.flips, relu_flips([self.masks[l]], [z + bias], [U * (z + bias).abs()]))
        self.st.append(s)

    def backward(self, g, grads):
        """g (rows, C_last): the gradient of the last activation with the device's decisions.  Fills
        grads[w|b|gamma|beta][l] = (value, bound) for l >= 1 and the BN / bias ones of layer 0; returns (dZ0, e_dZ0)"""
        n = self.rows_total or g.shape[0]
        fin = _store32 if self.store else (lambda v, e: e)
        eg = torch.zeros_like(g)
        for l in range(self.L - 1, -1, -1):
            s, d = self.st[l], self.layers[l]
            if self.bn:
                zc = self.zs[l].double() - s["mean"]
                x = zc * s["inv"]
                ed = _store32(zc, s["em32"])
                ex = _store32(x, ed * (s["inv"] + s["einv32"]) + zc.abs() * s["einv32"])
                del zc, ed
                ag, ax = g.abs() + eg, x.abs() + ex
                sg, sgx = g.sum(0), (g * x).sum(0)
                esg = eg.sum(0) + g64(n) * ag.sum(0)
                esgx = (eg * x.abs() + g.abs() * ex + eg * ex).sum(0) + g64(n) * (ag * ax).sum(0)
                grads["beta"][l] = (sg, _store32(sg, esg))
                grads["gamma"][l] = (sgx, _store32(sgx, esgx))
                mg0, mg1 = sg / n, sgx / n
                emg0, emg1 = _store32(mg0, esg / n), _store32(mg1, esgx / n)
                t = g - mg0 - x * mg1
                et = eg + emg0 + ex * (mg1.abs() + emg1) + x.abs() * emg1
                et = et + 3 * U * (ag + mg0.abs() + emg0 + ax * (mg1.abs() + emg1))
                a, ea = s["a"], s["ea32"]
                dz = a * t
                edz = _store32(dz, ea * (t.abs() + et) + a.abs() * et)
                del x, ex, ag, ax, t, et
            else:
                sg = g.sum(0)
                grads["b"][l] = (sg, fin(sg, eg.sum(0) + g64(n) * (g.abs() + eg).sum(0)))
                dz, edz = g, eg
            if l == 0:
                return dz, edz
            a_in = self.act(l - 1)
            w = d["w"]
            chunk, parts = wsplit(n, w.shape[0], w.shape[1])
            grads["w"][l] = weight_grad(dz, edz, a_in, U * a_in, chunk, parts, self.store)
            da, eda, _ = gemm(dz, edz, w, 0, w.shape[0])
            mk = self.masks[l - 1].to(da.dtype)
            g, eg = da * mk, eda * mk
            del da, eda, dz, edz


def _grads(L):
    return {k: [None] * L for k in ("w", "b", "gamma", "beta")}


# ------------------------------------------------------------------------------------------------ SA scale
def sa_rows0(xyz, centres, feats, idx, dev):
    """layer 0's rows in float64 and their bound: the xyz columns are fl32(xyz - centre) on the device"""
    xyz, centres, idx = xyz.to(dev).double(), centres.to(dev).double(), idx.to(dev).long()
    bi = torch.arange(idx.shape[0], device=dev)[:, None, None]
    rel = (xyz[bi, idx] - centres[:, :, None, :]).reshape(-1, 3)
    cols, ecols = [rel], [U * rel.abs()]
    if feats is not None:
        f = feats.detach().to(dev).double().transpose(1, 2)[bi, idx].reshape(-1, feats.shape[1])
        cols.append(f)
        ecols.append(torch.zeros_like(f))
    return torch.cat(cols, 1), torch.cat(ecols, 1)


def sa_scale(xyz, centres, feats, idx, layers, zs, stats, chosen, grad_out=None, dev="cpu", rows_total=None, store=True):
    """one SA scale replayed from the device's saved Z (per layer (rows, C_l)), statistics (per layer (4, C_l)) and chosen
    samples ((B * P, C_last)).  xyz (B, N, 3), centres (B, P, 3), feats (B, C, N) or None, idx (B, P, ns), grad_out
    (B, C_last, P).  -> Stack (its checks: every Z, statistic and running statistic; `out` (B, C_last, P); `pool`: the
    chosen samples' decision ratio and how many are not the first of identical rows) with, given grad_out, st.grads
    (w, b, gamma, beta per layer (value, bound)) and st.feats (sum, err, magnitude, count) of the feature scatter.
    rows_total / store: a bias chain replayed a group of scenes at a time (see Stack)"""
    B, P, ns = idx.shape
    a0, ea0 = sa_rows0(xyz, centres, feats, idx, dev)
    st = Stack(layers, zs, stats, dev, rows_total, store)
    w0 = st.layers[0]["w"]
    z0, ez0, _ = gemm(a0, ea0, w0.t(), 0, w0.shape[1])
    st.forward(z0, ez0)
    del z0, ez0
    last = st.act(st.L - 1)
    C = last.shape[1]
    out = last.view(B * P, ns, C).max(1).values
    st.out = (out.view(B, P, C).transpose(1, 2), U * out.view(B, P, C).transpose(1, 2))
    del last
    pre_dev = st.stats[-1][2] * st.zs[-1].double() + st.stats[-1][3]
    st.pool = pool_choices(chosen, pre_dev, 2 * U * pre_dev.abs(), a0, ns)
    del pre_dev
    if grad_out is None:
        return st
    rows = B * P * ns
    go = grad_out.to(dev).double().transpose(1, 2).reshape(B * P, C)
    g = torch.zeros(B * P, ns, C, dtype=torch.float64, device=dev)
    g.scatter_(1, chosen.to(dev).long().unsqueeze(1), go.unsqueeze(1))
    g = g.view(rows, C) * st.masks[-1].double()
    grads = _grads(st.L)
    dz0, edz0 = st.backward(g, grads)
    del g
    chunk, parts = wsplit(rows_total or rows, w0.shape[0], w0.shape[1])
    grads["w"][0] = weight_grad(dz0, edz0, a0, ea0, chunk, parts, store)
    st.grads = grads
    st.feats = None
    if feats is not None:
        da, eda, _ = gemm(dz0, edz0, w0, 0, w0.shape[0])
        v, ev = da[:, 3:], eda[:, 3:]
        c_feat, N = feats.shape[1], xyz.shape[1]
        point = (idx.to(dev).long() + torch.arange(B, device=dev)[:, None, None] * N).reshape(-1)
        acc = [torch.zeros(B * N, c_feat, dtype=torch.float64, device=dev).index_add_(0, point, t) for t in (v, ev, v.abs() + ev)]
        cnt = torch.zeros(B * N, dtype=torch.float64, device=dev).index_add_(0, point, torch.ones_like(point, dtype=torch.float64))
        st.feats = tuple(t.view(B, N, c_feat).transpose(1, 2) for t in acc) + (cnt.view(B, N),)
    return st


def finish_grads(parts):
    """the parameter gradients of a bias chain replayed in parts (Stack with store=False): {w, b: [(value, bound)]}
    summed over the parts, with the fp32 store of the device's result"""
    out = {}
    for k in ("w", "b"):
        out[k] = []
        for l in range(len(parts[0][k])):
            if parts[0][k][l] is None:
                out[k].append(None)
                continue
            v = sum(p[k][l][0] for p in parts)
            out[k].append((v, _store32(v, sum(p[k][l][1] for p in parts))))
    return out


def feats_grad(parts):
    """the feature gradient of several scales scattered into one buffer: (value, bound) from their Stack.feats"""
    v = sum(p[0] for p in parts)
    e = sum(p[1] for p in parts)
    mag = sum(p[2] for p in parts)
    cnt = sum(p[3] for p in parts)
    return v, e + gsum(cnt)[:, None, :] * mag


# ------------------------------------------------------------------------------------------------ FP module
def fp_module(known, skip, idx, w, layers, zs, stats, grad_out=None, dev="cpu"):
    """one FP module replayed from the device's saved Z and statistics, layer 0 projected as the device runs it.  known
    (B, ci, m), skip (B, cs, n) or None, idx / w (B, n, 3) the taps, grad_out (B, C_last, n).
    -> Stack (checks, `out` (B, C_last, n)) with, given grad_out, st.grads and st.known / st.skip (value, bound)"""
    B, ci, m = known.shape
    n = idx.shape[1]
    rows = B * n
    F = known.detach().to(dev).double().transpose(1, 2).reshape(B * m, ci)
    S = skip.detach().to(dev).double().transpose(1, 2).reshape(rows, -1) if skip is not None else None
    cs = 0 if S is None else S.shape[1]
    st = Stack(layers, zs, stats, dev)
    W0 = st.layers[0]["w"]
    Wi, Ws = W0[:, :ci], W0[:, ci:]
    c1 = W0.shape[0]
    P, eP, _ = gemm(F, 0, Wi.t(), 0, ci)
    idx, wt = idx.to(dev).long(), w.to(dev).double()
    tap = (idx + torch.arange(B, device=dev)[:, None, None] * m).reshape(rows, 3)
    wr = wt.reshape(rows, 3, 1)
    z0 = torch.zeros(rows, c1, dtype=torch.float64, device=dev)
    ez0 = torch.zeros_like(z0)
    for k in range(3):
        Pk, ePk = P[tap[:, k]], eP[tap[:, k]]
        z0 += wr[:, k] * Pk
        ez0 += wr[:, k] * ePk + 3 * U * (1 + 2 * U) * wr[:, k] * (Pk.abs() + ePk)
        del Pk, ePk
    if cs:
        zs_, ezs, _ = gemm(S, 0, Ws.t(), 0, cs)
        z0 += zs_
        ez0 += ezs
        del zs_, ezs
        ez0 = _store32(z0, ez0)
    st.forward(z0, ez0)
    del z0, ez0, P, eP
    last = st.act(st.L - 1)
    C = last.shape[1]
    last = last.view(B, n, C).transpose(1, 2)
    st.out = (last, U * last)
    if grad_out is None:
        return st
    g = grad_out.to(dev).double().transpose(1, 2).reshape(rows, C) * st.masks[-1].double()
    grads = _grads(st.L)
    dz0, edz0 = st.backward(g, grads)
    del g
    # G = I^T dZ0, an fma chain per known point
    flat = tap.reshape(-1)
    G = torch.zeros(B * m, c1, dtype=torch.float64, device=dev)
    eG, mag = torch.zeros_like(G), torch.zeros_like(G)
    for k in range(3):
        wd, ewd = wr[:, k] * dz0, wr[:, k] * edz0
        G.index_add_(0, tap[:, k], wd)
        eG.index_add_(0, tap[:, k], ewd)
        mag.index_add_(0, tap[:, k], wd.abs() + ewd)
        del wd, ewd
    cnt = torch.zeros(B * m, dtype=torch.float64, device=dev).index_add_(0, flat, torch.ones_like(flat, dtype=torch.float64))[:, None]
    eG += cnt * U / (1 - cnt * U) * mag
    del mag
    chunk_i, parts_i = wsplit(B * m, c1, ci)
    dwi, edwi = weight_grad(G, eG, F, 0, chunk_i, parts_i)
    dF, edF, _ = gemm(G, eG, Wi, 0, c1)
    st.known = (dF.view(B, m, ci).transpose(1, 2), edF.view(B, m, ci).transpose(1, 2))
    st.skip = None
    if cs:
        chunk0, parts0 = wsplit(rows, c1, max(cs, 1))
        dws, edws = weight_grad(dz0, edz0, S, 0, chunk0, parts0)
        dS, edS, _ = gemm(dz0, edz0, Ws, 0, c1)
        st.skip = (dS.view(B, n, cs).transpose(1, 2), edS.view(B, n, cs).transpose(1, 2))
        grads["w"][0] = (torch.cat([dwi, dws], 1), torch.cat([edwi, edws], 1))
    else:
        grads["w"][0] = (dwi, edwi)
    st.grads = grads
    return st


# ------------------------------------------------------------------------------------------------ checks
def ratio(got, ref, bound):
    """largest |got - ref| / bound (0 where both are equal; inf where got is not finite or the bound is 0 and they differ)"""
    got = got.to(ref.device).double()
    err = (got - ref).abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / bound)
    r = torch.where(torch.isfinite(got), r, torch.full_like(r, math.inf))
    return float(r.max()) if r.numel() else 0.0


def relu_flips(masks, pre, e_pre):
    """largest |pre| / e_pre over the elements whose device ReLU decision differs from the reference's sign (<= 1: every
    flip lies within the bound of zero)"""
    worst = 0.0
    for mk, p, e in zip(masks, pre, e_pre):
        flip = mk.to(p.device) != (p > 0)
        if flip.any():
            worst = max(worst, float((p[flip].abs() / e[flip]).max()))
    return worst


def pool_choices(chosen, pre, e_pre, a0, ns):
    """the device's chosen samples against the reference's pre-activations of the last layer: (largest shortfall of the
    chosen value below the group's maximum over the sum of the two bounds, number of choices that are not the first of
    the group's bitwise identical rows).  A device that keeps the first maximum must take the first of identical rows:
    identical rows give identical values."""
    C = pre.shape[1]
    p = pre.view(-1, ns, C)
    e = e_pre.view(-1, ns, C)
    ch = chosen.to(p.device).long()
    pc = p.gather(1, ch.unsqueeze(1)).squeeze(1)
    ec = e.gather(1, ch.unsqueeze(1)).squeeze(1)
    short = (p.max(1).values - pc).clamp_min(0)
    worst = float((short / (ec + e.max(1).values)).max()) if short.numel() else 0.0
    key = torch.rand(a0.shape[1], generator=torch.Generator().manual_seed(0), dtype=torch.float64).to(a0.device) + 0.5
    h = (a0 @ key).view(-1, ns)                           # equal rows hash equal; unequal ones differ but by a fluke
    first = (h[:, :, None] == h[:, None, :]).float().argmax(-1)          # (groups, ns): the first identical sample
    not_first = int((first.gather(1, ch) != ch).sum())
    return worst, not_first


# ------------------------------------------------------------------------------------------------ fp32 emulation
# An fp32 model of the kernels' rounding points, to show on the CPU that the bound holds for plausible accumulation
# orders and that it catches subtle mistakes.  Each mutant plants one:
SA_MUTANTS = ("no_sum_g", "no_sum_gx", "unbiased_norm", "biased_running", "wrong_pool", "no_relu_mask",
              "no_sum_gx_small_gamma",   # no_sum_gx on the channels with |gamma| < 1e-2 only
              "drop_xyz_grad",           # layer 0's weight gradient of the xyz-offset columns dropped
              "pool_last_max")           # the pooled gradient sent to the last maximal sample instead of the first
FP_MUTANTS = ("no_bn_term", "unbiased_norm", "no_relu_mask", "wrong_tap", "swap_cols",
              "skip_off_by_one")         # the skip gradient of channel k written to channel k + 1
ORDERS = ("sequential", "reversed", "pairwise8")


def tf32(x):
    """cvt.rn.tf32.f32 of an fp32 CPU tensor (mlp_reference.tf32_rn)"""
    return torch.from_numpy(tf32_rn(x.float().contiguous().numpy()))


def mm32(X, Y, order):
    """X @ Y from TF32 operands with an fp32 accumulator over K in `order` (products of TF32 values are exact in fp32)"""
    X, Y = tf32(X), tf32(Y)
    K = X.shape[1]
    acc = torch.zeros(X.shape[0], Y.shape[1])
    if order == "pairwise8":
        pad = -K % 8
        X, Y = torch.nn.functional.pad(X, (0, pad)), torch.nn.functional.pad(Y, (0, 0, 0, pad))
        for k0 in range(0, K + pad, 8):
            q = X[:, k0:k0 + 8, None] * Y[None, k0:k0 + 8, :]
            while q.shape[1] > 1:
                q = q[:, 0::2] + q[:, 1::2]
            acc = acc + q[:, 0]
        return acc
    for k in (range(K) if order == "sequential" else range(K - 1, -1, -1)):
        acc = acc + X[:, k:k + 1] * Y[k:k + 1]
    return acc


def _dw32(dz, a, order):
    """dW = dZ^T A: fp32 partials over the row chunks of the device's split, summed in float64, stored as fp32"""
    chunk, _ = wsplit(dz.shape[0], dz.shape[1], a.shape[1])
    s = torch.zeros(dz.shape[1], a.shape[1], dtype=torch.float64)
    for r0 in range(0, dz.shape[0], chunk):
        s += mm32(dz[r0:r0 + chunk].t(), a[r0:r0 + chunk], order).double()
    return s.float()


def _fma(a, b, c):
    return (a.double() * b.double() + c.double()).float()


class _EmuStack:
    """the layer stack in fp32 as sa_train.cu runs it"""

    def __init__(self, layers, order, mutant):
        self.layers, self.order, self.mutant = layers, order, mutant
        self.bn = "gamma" in layers[0]
        self.st, self.running = [], []

    def layer(self, l, z):
        d = self.layers[l]
        n = z.shape[0]
        if self.bn:
            z64 = z.double()
            mean = z64.sum(0) / n
            var = ((z64 * z64).sum(0) / n - mean * mean).clamp_min(0)
            var_norm = var * n / (n - 1) if self.mutant == "unbiased_norm" else var
            inv = 1.0 / torch.sqrt(var_norm + d["eps"])
            ga, be, m = d["gamma"], d["beta"], d["momentum"]
            a, b = (ga * inv).float(), (be - mean * ga * inv).float()
            rv = var if self.mutant == "biased_running" else var * n / (n - 1)
            self.running.append((((1 - m) * d["rm"] + m * mean).float(), ((1 - m) * d["rv"] + m * rv).float()))
            s = dict(z=z, mean=mean.float(), inv=inv.float(), a=a, b=b, gamma=ga)
        else:
            s = dict(z=z, mean=torch.zeros(z.shape[1]), inv=torch.ones(z.shape[1]), a=torch.ones(z.shape[1]),
                     b=d["b"].float() if d["b"] is not None else torch.zeros(z.shape[1]))
        s["stats"] = torch.stack([s["mean"], s["inv"], s["a"], s["b"]])
        pre = _fma(s["a"], z, s["b"])
        s["mask"] = pre > 0
        self.st.append(s)
        return pre

    def forward(self, z0):
        self.inputs = []
        pre = self.layer(0, z0)
        for l in range(1, len(self.layers)):
            act = pre.clamp_min(0)
            self.inputs.append(act)
            pre = self.layer(l, mm32(act, self.layers[l]["w"].float().t(), self.order))
        return pre

    def backward(self, g, grads):
        n = g.shape[0]
        for l in range(len(self.layers) - 1, -1, -1):
            s, d = self.st[l], self.layers[l]
            if self.bn:
                x = (s["z"] - s["mean"]) * s["inv"]
                sg, sgx = g.double().sum(0), (g.double() * x.double()).sum(0)
                grads["beta"][l], grads["gamma"][l] = sg.float(), sgx.float()
                mg0, mg1 = (sg / n).float(), (sgx / n).float()
                if self.mutant == "no_sum_g":
                    mg0 = torch.zeros_like(mg0)
                if self.mutant in ("no_sum_gx", "no_bn_term"):
                    mg1 = torch.zeros_like(mg1)
                if self.mutant == "no_sum_gx_small_gamma":
                    mg1 = torch.where(s["gamma"].abs() < 1e-2, torch.zeros_like(mg1), mg1)
                dz = s["a"] * ((g - mg0) - x * mg1)
            else:
                grads["b"][l] = g.double().sum(0).float()
                dz = g
            if l == 0:
                return dz
            grads["w"][l] = _dw32(dz, self.inputs[l - 1], self.order)
            g = mm32(dz, d["w"].float(), self.order)
            if self.mutant != "no_relu_mask":
                g = g * self.st[l - 1]["mask"]


def _scatter_order(rows, order, seed):
    if order == "sequential":
        return torch.arange(rows)
    if order == "reversed":
        return torch.arange(rows - 1, -1, -1)
    return torch.randperm(rows, generator=torch.Generator().manual_seed(seed))      # atomics: any order


def emulate_sa(xyz, centres, feats, idx, layers, grad_out, order="sequential", mutant=None, grad_feats=None):
    """one SA scale in fp32 -> dict(out (B, C, P), running, masks, chosen, w, b, gamma, beta); the feature gradient is
    scattered (fp32, in an order that depends on `order`) into grad_feats (B, c_feat, N), which the caller owns"""
    B, P, ns = idx.shape
    N = xyz.shape[1]
    idx = idx.long()
    bi = torch.arange(B)[:, None, None]
    a0 = (xyz[bi, idx] - centres[:, :, None, :]).reshape(-1, 3)
    if feats is not None:
        a0 = torch.cat([a0, feats.transpose(1, 2)[bi, idx].reshape(-1, feats.shape[1])], 1)
    st = _EmuStack(layers, order, mutant)
    pre = st.forward(mm32(a0, layers[0]["w"].float().t(), order)).view(B * P, ns, -1)
    best, arg = pre[:, 0].clone(), torch.zeros(pre.shape[0], pre.shape[2], dtype=torch.long)
    for s in range(1, ns):
        v = pre[:, s]
        take = (v < best) if mutant == "wrong_pool" else (v >= best) if mutant == "pool_last_max" else (v > best)
        best, arg = torch.where(take, v, best), torch.where(take, torch.full_like(arg, s), arg)
    C = pre.shape[2]
    out = best.clamp_min(0).view(B, P, C).transpose(1, 2)
    go = grad_out.transpose(1, 2).reshape(B * P, C)
    g = torch.zeros(B * P, ns, C).scatter_(1, arg.unsqueeze(1), go.unsqueeze(1)).view(-1, C)
    if mutant != "no_relu_mask":
        g = g * st.st[-1]["mask"]
    grads = _grads(len(layers))
    dz0 = st.backward(g, grads)
    grads["w"][0] = _dw32(dz0, a0, order)
    if mutant == "drop_xyz_grad":
        grads["w"][0][:, :3] = 0
    if feats is not None:
        v = mm32(dz0, layers[0]["w"].float(), order)[:, 3:]
        point = (idx + bi * N).reshape(-1)
        perm = _scatter_order(point.numel(), order, seed=ns)
        flat = grad_feats.transpose(1, 2).reshape(B * N, -1).contiguous()
        flat.index_add_(0, point[perm], v[perm])
        grad_feats.copy_(flat.view(B, N, -1).transpose(1, 2))
    return dict(out=out, running=st.running, z=[s["z"] for s in st.st], stats=[s["stats"] for s in st.st], chosen=arg, **grads)


def emulate_fp(known, skip, idx, w, layers, grad_out, order="sequential", mutant=None):
    """one FP module in fp32, layer 0 projected -> dict(out, running, masks, w, b, gamma, beta, known, skip)"""
    B, ci, m = known.shape
    n = idx.shape[1]
    rows = B * n
    F = known.transpose(1, 2).reshape(B * m, ci)
    W0 = layers[0]["w"].float()
    Wi, Ws = W0[:, :ci], W0[:, ci:]
    if mutant == "swap_cols":
        Wi, Ws = W0[:, W0.shape[1] - ci:], W0[:, :W0.shape[1] - ci]
    P = mm32(F, Wi.t(), order)
    taps = (idx.long() + torch.arange(B)[:, None, None] * m).reshape(rows, 3)
    if mutant == "wrong_tap":
        taps = taps[:, [1, 0, 2]]
    wr = w.reshape(rows, 3)
    z0 = _fma(wr[:, 2:3], P[taps[:, 2]], _fma(wr[:, 0:1], P[taps[:, 0]], wr[:, 1:2] * P[taps[:, 1]]))
    S = skip.transpose(1, 2).reshape(rows, -1) if skip is not None else None
    if S is not None:
        z0 = mm32(S, Ws.t(), order) + z0
    st = _EmuStack(layers, order, mutant)
    pre = st.forward(z0)
    C = pre.shape[1]
    out = pre.clamp_min(0).view(B, n, C).transpose(1, 2)
    g = grad_out.transpose(1, 2).reshape(rows, C)
    if mutant != "no_relu_mask":
        g = g * st.st[-1]["mask"]
    grads = _grads(len(layers))
    dz0 = st.backward(g, grads)
    G = torch.zeros(B * m, dz0.shape[1])
    for q in _scatter_order(rows * 3, order, seed=1).tolist():       # an fma per reference, in list order
        r, t = divmod(q, 3)
        G[taps[r, t]] = _fma(wr[r, t], dz0[r], G[taps[r, t]])
    dwi = _dw32(G, F, order)
    dF = mm32(G, Wi, order)
    res = dict(out=out, running=st.running, z=[s["z"] for s in st.st], stats=[s["stats"] for s in st.st],
               known=dF.view(B, m, ci).transpose(1, 2))
    if S is not None:
        dS = mm32(dz0, Ws, order)
        if mutant == "skip_off_by_one":
            dS = torch.roll(dS, 1, 1)
        res["skip"] = dS.view(B, n, -1).transpose(1, 2)
        grads["w"][0] = torch.cat([dwi, _dw32(dz0, S, order)], 1)
    else:
        grads["w"][0] = dwi
    res.update(grads)
    return res


# ------------------------------------------------------------------------------------------------ comparisons
def ratios(got, st, feats=None):
    """{quantity: largest error / bound}: the Stack's checks (every Z and statistic), and what `got` (out, running
    [(rm, rv)], w / b / gamma / beta per layer, known / skip) shares with it; feats: (device, (value, bound)) of SA"""
    out = {k: ratio(*v) for k, v in st.checks.items()}
    out["out"] = ratio(got["out"], *st.out)
    for l, (g, s) in enumerate(zip(got.get("running", []), st.st)):
        if s["running"] is not None:
            r = s["running"]
            out["running_mean%d" % l] = ratio(g[0], r[0], r[1])
            out["running_var%d" % l] = ratio(g[1], r[2], r[3])
    for k in ("w", "b", "gamma", "beta"):
        for l, (g, r) in enumerate(zip(got.get(k, []), getattr(st, "grads", {}).get(k, []))):
            if g is not None and r is not None:
                out["%s%d" % (k, l)] = ratio(g.reshape(r[0].shape), r[0], r[1])
    for k in ("known", "skip"):
        if got.get(k) is not None and getattr(st, k, None) is not None:
            out[k] = ratio(got[k], *getattr(st, k))
    if feats is not None:
        out["feats"] = ratio(feats[0], *feats[1])
    return out


def _fwd_tol(g, r):
    return float((g.double().to(r.device) - r).abs().max() / (2e-3 * r.abs().max().clamp_min(1e-30)))


def _grad_tol(g, r):
    d = g.double().to(r.device) - r
    return max(float(d.abs().max() / (5e-3 * r.abs().max().clamp_min(1e-30))), float(d.norm() / (2e-3 * r.norm().clamp_min(1e-30))))


def old_ratios(got, st, feats=None):
    """the same outputs and gradients under the tensor-wide tolerances of sa_train_reference / fp_train_reference: forward
    within 2e-3 max|ref|, gradients within 5e-3 max|ref| and 2e-3 relative Frobenius (<= 1 passes)"""
    out = {"out": _fwd_tol(got["out"], st.out[0])}
    for l, (g, s) in enumerate(zip(got.get("running", []), st.st)):
        if s["running"] is not None:
            r = s["running"]
            out["running_mean%d" % l] = float((g[0].double().to(r[0].device) - r[0]).abs().max()
                                              / (2e-3 * torch.maximum(r[0].abs().max(), r[2].clamp_min(0).sqrt().max())))
            out["running_var%d" % l] = _fwd_tol(g[1], r[2])
    for k in ("w", "b", "gamma", "beta"):
        for l, (g, r) in enumerate(zip(got.get(k, []), getattr(st, "grads", {}).get(k, []))):
            if g is not None and r is not None:
                out["%s%d" % (k, l)] = _grad_tol(g.reshape(r[0].shape), r[0])
    for k in ("known", "skip"):
        if got.get(k) is not None and getattr(st, k, None) is not None:
            out[k] = _grad_tol(got[k], getattr(st, k)[0])
    if feats is not None:
        out["feats"] = _grad_tol(feats[0], feats[1][0])
    return out


def old_pool_check(chosen, st, ns):
    """the tensor-wide tests' decision check: a chosen sample within 2e-3 max|y| of its group's maximum (<= 1 passes)"""
    y = st.act(st.L - 1)
    y = y.view(-1, ns, y.shape[1])
    picked = y.gather(1, chosen.to(y.device).long().unsqueeze(1)).squeeze(1)
    return float((y.max(1).values - picked).max() / (2e-3 * y.abs().max()))
