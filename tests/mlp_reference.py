"""A float64 reference of the wgmma MLP chain (csrc/mlp_tc.cu) with a rigorous per-element error bound.

The tensor core's fp32 accumulation order and rounding are not specified, so no host model can match the kernel bit for
bit.  Instead the reference computes every layer in float64 from exactly the TF32 operands the tensor core sees, and
carries a bound on |kernel - reference| per output element:

  weights     read back from the packed image (unpack(), written from the K-major SWIZZLE_128B layout, not from the
              packer), so they are the TF32 values the kernel multiplies, in the caller's column order
  layer 0     the operand is emulated exactly where the kernel's arithmetic is plain IEEE fp32: SA rows are
              tf32_rn(float32(x - cx)) and tf32_rn(features), direct rows and FP skip channels tf32_rn(input).  The FP
              interpolation fma(w2,p2, fma(w0,p0, w1*p1)) is bounded instead: 3 fp32 roundings of sum |w_k p_k|, then a
              TF32 half-ulp
  a layer     z = W a (float64), y = s z + t (t alone when the scale is folded into W), ReLU unless it is the linear
              last layer; inner activations stay unrounded in the reference
  the bound   accumulation  GAMMA(K) * |W| (|a| + e) + |W| e      (e: the bound on the layer's input)
              epilogue      one fp32 rounding of s z + t
              ReLU, max     1-Lipschitz: the bound passes through (max-pooled bounds for the SA max)
              TF32 rounding a half-ulp, 2^-11 |value|, wherever the kernel rounds an activation: between the layers of a
                            launch and on the intermediate rows of a split chain

The check is |got - ref| <= bound for every element.  emulate() is an fp32 model of the kernel's rounding points (used to
show, without a GPU, that the bound holds for plausible accumulation orders and that it catches subtle mistakes).
"""
import numpy as np

from pointrcnn_b200 import mlp_chain

KC = 32                       # K columns per chunk of the packed image (one 128-byte swizzle row)
U32 = 2.0 ** -24              # unit roundoff of one fp32 round-to-nearest
TF32_HALF_ULP = 2.0 ** -11    # relative half-ulp of a round-to-nearest to TF32 (10 stored mantissa bits)


def gamma(k_pad):
    """Accumulation error of a K-term dot product, relative to sum |w_k a_k|.  The products of TF32 operands are exact in
    fp32; wgmma adds them in fp32 in an order and with a rounding that are not documented.  ASSUMPTION: each of the K_pad
    additions (plus the alignment of the running sum across K=8 steps and chunks) loses at most two fp32 ulps, i.e.
    2^-22 of the magnitude summed so far, and that magnitude never exceeds sum |w_k a_k|."""
    return (k_pad + 2) * 2.0 ** -22


def round_up(a, b):
    return (a + b - 1) // b * b


# ------------------------------------------------------------------------------------------------ TF32 roundings
def tf32_rn(x):
    """cvt.rn.tf32.f32: round to nearest, ties to even (the kernel's activations and gathered operands)"""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    finite = (u & 0x7F800000) != 0x7F800000
    r = (u + 0xFFF + ((u >> 13) & 1)) & 0xFFFFE000
    return np.where(finite, r, u).astype(np.uint32).view(np.float32)


def tf32_rna(x):
    """cvt.rna.tf32.f32: round to nearest, ties away from zero (the host packer)"""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).copy()
    finite = (u & 0x7F800000) != 0x7F800000
    u[finite] += 0x1000
    u &= 0xFFFFE000
    return u.view(np.float32)


# ------------------------------------------------------------------------------------------------ packed image
def k_order(kind, split, c_in):
    """Layer 0's K order in the packed image: caller column per K index, -1 for padding.  kind 0 (SA, split = c_feat): up to
    five feature channels ride with xyz in one segment [xyz, feats], more go first as their own segment [feats][xyz];
    kind 1 (FP, split = c_known): [interp][skip], two padded segments (one when there is no skip); kind 2: one segment."""
    if kind == 0:
        segs = [(0, 3 + split)] if split <= 5 else [(3, split), (0, 3)]
    elif kind == 1 and c_in > split:
        segs = [(0, split), (split, c_in - split)]
    else:
        segs = [(0, c_in)]
    cols = []
    for first, width in segs:
        cols += list(range(first, first + width)) + [-1] * (round_up(width, KC) - width)
    return np.array(cols, dtype=np.int64), [w for _, w in segs]


class Layer:
    """one layer read back from a packed image: W (c_out, k_in) in the caller's column order; Wk (np, k_pad) the tile rows in
    K order, kmap the caller column of every K index (-1: padding)"""

    def __init__(self, W, Wk, kmap):
        self.W, self.Wk, self.kmap = W, Wk, kmap
        self.k_pad = Wk.shape[1]


def unpack(img, kind, split, c_in, c_out):
    """The packed image back to per-layer weight matrices.  Element (kc, n, kk) of a layer's (np x k_pad) image sits at
    kc*np*32 + n*32 + (((kk >> 2) ^ (n & 7)) << 2) + (kk & 3): K-major rows of 128 bytes, 16-byte units XOR-swizzled by the
    row index.  Raises if an element that must be padding is not zero or the image has the wrong size."""
    layers, off = [], 0
    for l, co in enumerate(c_out):
        npad = round_up(co, 32)
        if l == 0:
            kmap, _ = k_order(kind, split, c_in)
            k_in = c_in
        else:
            k_in = c_out[l - 1]
            kmap = np.r_[np.arange(k_in), -np.ones(round_up(k_in, 32) - k_in, np.int64)]
        nch = len(kmap) // KC
        kc, n, kk = np.meshgrid(np.arange(nch), np.arange(npad), np.arange(KC), indexing="ij")
        pos = off + kc * npad * KC + n * KC + (((kk >> 2) ^ (n & 7)) << 2) + (kk & 3)
        assert pos.max() < img.size, "packed image too small"
        Wk = img[pos].transpose(1, 0, 2).reshape(npad, nch * KC)
        assert not Wk[co:].any() and not Wk[:, kmap < 0].any(), "layer %d: padding of the packed image is not zero" % l
        W = np.zeros((co, k_in), np.float32)
        W[:, kmap[kmap >= 0]] = Wk[:co, kmap >= 0]
        layers.append(Layer(W, Wk, kmap))
        off += nch * npad * KC
    assert off == img.size, "packed image has %d floats, the layers %d" % (img.size, off)
    return layers


# ------------------------------------------------------------------------------------------------ cases
class Chain:
    """weights / scale / shift of one chain and how it is packed.  scale None = folded (the descriptor's scale is NULL)."""

    def __init__(self, rng, kind, split, c_in, c_out, folded, linear):
        dims = [c_in] + list(c_out)
        self.kind, self.split, self.c_in, self.c_out, self.linear = kind, split, c_in, list(c_out), linear
        self.weights = [(rng.standard_normal((co, ci)) * np.sqrt(2.0 / ci)).astype(np.float32) for ci, co in zip(dims[:-1], dims[1:])]
        # unfolded scales take both signs (BN with negative gamma); a folded scale lives in the weights
        self.scale = None if folded else [(rng.uniform(0.5, 1.5, co) * rng.choice([-1.0, 1.0], co)).astype(np.float32) for co in c_out]
        self.shift = [rng.normal(0, 0.2, co).astype(np.float32) for co in c_out]

    def packed(self):
        img = mlp_chain.pack_image(self.kind, self.split, self.weights)
        return img, unpack(img, self.kind, self.split, self.c_in, self.c_out)


def sa_inputs(rng, b, n, npoint, ns, c_feat):
    """SA operands.  idx references only the even points of a scene: the odd rows of xyz and feats_pm are NaN, which the
    kernel must never read."""
    xyz = rng.uniform(-1, 1, (b, n, 3)).astype(np.float32)
    feats = rng.standard_normal((b, n, c_feat)).astype(np.float32)
    xyz[:, 1::2] = np.nan
    feats[:, 1::2] = np.nan
    return dict(xyz=xyz, feats_pm=feats, new_xyz=rng.uniform(-1, 1, (b, npoint, 3)).astype(np.float32),
                idx=(2 * rng.integers(0, (n + 1) // 2, (b, npoint, ns))).astype(np.int32))


def fp_inputs(rng, b, n, m, c_known, c_skip):
    """FP operands.  idx references only the even known points; the odd rows of known_pm are NaN."""
    known = rng.standard_normal((b, m, c_known)).astype(np.float32)
    known[:, 1::2] = np.nan
    w = rng.uniform(0.05, 1.0, (b, n, 3)).astype(np.float32)
    return dict(known_pm=known, idx=(2 * rng.integers(0, (m + 1) // 2, (b, n, 3))).astype(np.int32),
                weight=(w / w.sum(-1, keepdims=True)).astype(np.float32),
                skip=rng.standard_normal((b, c_skip, n)).astype(np.float32))


def rows_inputs(rng, rows, c_a, a_pitch, a_off, c_b, b_pitch, b_off):
    """row operands: segment a = columns [a_off, a_off + c_a) of a (rows, a_pitch) buffer, b likewise; every other column
    of the buffers is NaN (prb_mlp_rows2 must read only [:c_a] / [:c_b] of each row)"""
    A = np.full((rows, a_pitch), np.nan, np.float32)
    A[:, a_off:a_off + c_a] = rng.standard_normal((rows, c_a))
    out = dict(a=A, a_off=a_off, c_a=c_a)
    if c_b:
        B = np.full((rows, b_pitch), np.nan, np.float32)
        B[:, b_off:b_off + c_b] = rng.standard_normal((rows, c_b))
        out.update(b=B, b_off=b_off, c_b=c_b)
    return out


# ------------------------------------------------------------------------------------------------ layer 0
FP_INTERP_ROUNDINGS = 3 * U32 * (1 + 2 * U32)   # fl(w1 p1), then two fma roundings, of sum |w_k p_k| (second-order terms included)


def layer0(kind, inp, mutant=None):
    """Layer 0's operand in the caller's column order: (a, e) with a (rows, c_in) float64 and e its error bound (0: exact).
    SA rows are (scene, centre, sample) in order; FP rows (scene, point)."""
    if kind == "sa":
        xyz, new_xyz, idx, feats = inp["xyz"], inp["new_xyz"], inp["idx"], inp["feats_pm"]
        b, npoint, ns = idx.shape
        g = np.take_along_axis(xyz, idx.reshape(b, -1, 1).astype(np.int64), 1).reshape(b, npoint, ns, 3)
        centre = new_xyz
        if mutant == "rel_xyz_next_centre":
            centre = np.roll(new_xyz.reshape(-1, 3), -1, 0).reshape(new_xyz.shape)
        rel = tf32_rn((g - centre[:, :, None, :]).astype(np.float32))
        f = np.take_along_axis(feats, idx.reshape(b, -1, 1).astype(np.int64), 1).reshape(b, npoint, ns, -1)
        a = np.concatenate([rel, tf32_rn(f)], -1).reshape(b * npoint * ns, -1)
        return a.astype(np.float64), 0.0
    if kind == "fp":
        known, idx, w, skip = inp["known_pm"], inp["idx"], inp["weight"].astype(np.float64), inp["skip"]
        b, n, _ = idx.shape
        p = np.stack([np.take_along_axis(known, idx[:, :, k:k + 1].astype(np.int64), 1) for k in range(3)], 2).astype(np.float64)
        if mutant == "fp_weights_swapped":
            w = w[:, :, [1, 0, 2]]
        prod = w[..., None] * p                    # (b, n, 3, c_known), each product exact in float64
        v = prod.sum(2)
        e = FP_INTERP_ROUNDINGS * np.abs(prod).sum(2)
        e = e + TF32_HALF_ULP * (np.abs(v) + e)   # the gathered value is rounded to TF32
        s = np.ascontiguousarray(skip.transpose(0, 2, 1))
        if mutant == "skip_transposed" and s.shape[2] >= 2:
            s = s[:, :, [1, 0] + list(range(2, s.shape[2]))]
        a = np.concatenate([v, tf32_rn(s).astype(np.float64)], -1).reshape(b * n, -1)
        e = np.concatenate([e, np.zeros(s.shape)], -1).reshape(b * n, -1)
        return a, e
    x = inp["a"][:, inp["a_off"]:inp["a_off"] + inp["c_a"]]
    if "b" in inp:
        x = np.concatenate([x, inp["b"][:, inp["b_off"]:inp["b_off"] + inp["c_b"]]], 1)
    return tf32_rn(x).astype(np.float64), 0.0


# ------------------------------------------------------------------------------------------------ reference and bound
def reference(chain, layers, a, e):
    """float64 chain over layer-0 rows: (y, bound) of the last layer per row, padded to its np channels (the padding
    channels are exactly 0, bound 0)"""
    L = len(layers)
    for l, ly in enumerate(layers):
        Wa = np.abs(ly.W).astype(np.float64)
        z = a @ ly.W.T.astype(np.float64)
        ez = gamma(ly.k_pad) * ((np.abs(a) + e) @ Wa.T)
        if np.ndim(e):
            ez += e @ Wa.T
        s = 1.0 if chain.scale is None else chain.scale[l].astype(np.float64)
        y = z * s + chain.shift[l]
        ey = np.abs(s) * ez
        ey = ey + U32 * (np.abs(y) + ey)                        # one fp32 rounding of s z + t
        last = l == L - 1
        if not (last and chain.linear):
            y = np.maximum(y, 0)
        if not last:
            ey = ey + TF32_HALF_ULP * (np.abs(y) + ey)          # the activation is rounded to TF32
        a, e = y, ey
    npad = round_up(chain.c_out[-1], 32)
    pad = ((0, 0), (0, npad - a.shape[1]))
    return np.pad(a, pad), np.pad(e, pad)


def pool(y, ns):
    """max over the samples of a centre: rows (centres * ns, c) -> (centres, c)"""
    return y.reshape(-1, ns, y.shape[1]).max(1)


def expected(kind, chain, layers, inp):
    """(reference, bound) in the kernel's output layout: SA (b, c_last, npoint), FP (b, c_last, n), rows (rows, np_last)"""
    a, e = layer0(kind, inp)
    y, ey = reference(chain, layers, a, e)
    C = chain.c_out[-1]
    if kind == "sa":
        b, npoint, ns = inp["idx"].shape
        return [np.ascontiguousarray(pool(v, ns)[:, :C].reshape(b, npoint, C).transpose(0, 2, 1)) for v in (y, ey)]
    if kind == "fp":
        b, n, _ = inp["idx"].shape
        return [np.ascontiguousarray(v[:, :C].reshape(b, n, C).transpose(0, 2, 1)) for v in (y, ey)]
    return y, ey


def check(got, ref, bound):
    """(every element inside its bound, max err / bound, number outside).  NaN or Inf in `got` is outside."""
    err = np.abs(got.astype(np.float64) - ref)
    ok = err <= bound
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = np.where(err == 0, 0.0, err / bound)
    ratio = np.where(np.isfinite(got), ratio, np.inf)
    return bool(ok.all()), float(np.nanmax(ratio)) if ratio.size else 0.0, int((~ok).sum())


# ------------------------------------------------------------------------------------------------ fp32 emulation
ORDERS = ("sequential", "reversed", "pairwise8")
MUTANTS = ("drop_partial_kstep", "shift_off_by_one", "skip_transposed", "fp_weights_swapped", "rel_xyz_next_centre",
           "pool_neighbour_sample", "carry_leak", "relu_on_linear")


def _chunk_sum(P, order):
    """fp32 sum over the last axis (32 products of one K chunk) in the given order"""
    f = np.float32
    if order == "sequential":
        s = P[..., 0]
        for k in range(1, P.shape[-1]):
            s = (s + P[..., k]).astype(f)
        return s
    if order == "reversed":
        s = P[..., -1]
        for k in range(P.shape[-1] - 2, -1, -1):
            s = (s + P[..., k]).astype(f)
        return s
    steps = []
    for k0 in range(0, P.shape[-1], 8):       # a pairwise tree per K=8 step, the steps added in K order
        q = P[..., k0:k0 + 8]
        while q.shape[-1] > 1:
            q = (q[..., 0::2] + q[..., 1::2]).astype(f)
        steps.append(q[..., 0])
    s = steps[0]
    for t in steps[1:]:
        s = (s + t).astype(f)
    return s


def _fma32(a, s, t):
    return (a.astype(np.float64) * s + t).astype(np.float32)


def emulate(kind, chain, layers, inp, order="sequential", mutant=None):
    """fp32 model of the kernel: layer-0 operand as gathered (FP interpolation with the kernel's fma contraction), per layer
    fp32 accumulation chunk by chunk in K order (the chunk's products summed in `order`), epilogue fma in fp32, ReLU +
    TF32 rounding between layers, the SA max-pool.  `mutant` plants one subtle mistake.  Same layout as expected()."""
    f = np.float32
    if kind == "fp":
        known, idx, w, skip = inp["known_pm"], inp["idx"], inp["weight"], inp["skip"]
        b, n, _ = idx.shape
        p = [np.take_along_axis(known, idx[:, :, k:k + 1].astype(np.int64), 1) for k in range(3)]
        w0, w1, w2 = (w[:, :, k:k + 1] for k in range(3))
        if mutant == "fp_weights_swapped":
            w0, w1 = w1, w0
        v = _fma32(p[2], w2.astype(np.float64), _fma32(p[0], w0.astype(np.float64), (w1 * p[1]).astype(f)))
        s = np.ascontiguousarray(skip.transpose(0, 2, 1))
        if mutant == "skip_transposed" and s.shape[2] >= 2:
            s = s[:, :, [1, 0] + list(range(2, s.shape[2]))]
        a = tf32_rn(np.concatenate([v, s], -1).reshape(b * n, -1))
    else:
        a = layer0(kind, inp, mutant)[0].astype(f)
    L = len(layers)
    for l, ly in enumerate(layers):
        A = np.zeros((a.shape[0], ly.k_pad), f)
        A[:, ly.kmap >= 0] = a[:, ly.kmap[ly.kmap >= 0]]
        if l == 0 and mutant == "drop_partial_kstep":
            # the last K=8 step with data of every segment that ends inside a chunk is skipped
            _, widths = k_order(chain.kind, chain.split, chain.c_in)
            k0 = 0
            for wdt in widths:
                if wdt % KC:
                    last = k0 + (wdt // 8 if wdt % 8 else wdt // 8 - 1) * 8
                    A[:, last:last + 8] = 0
                k0 += round_up(wdt, KC)
        npad = ly.Wk.shape[0]
        acc = np.zeros((a.shape[0], npad), f)
        for c0 in range(0, ly.k_pad, KC):
            P = A[:, None, c0:c0 + KC] * ly.Wk[None, :, c0:c0 + KC]      # exact: TF32 x TF32 fits fp32
            acc = (acc + _chunk_sum(P, order)).astype(f)
        sh = np.pad(chain.shift[l], (0, npad - chain.c_out[l]))
        if mutant == "shift_off_by_one":
            sh = np.r_[sh[1:], 0].astype(f)
        sc = np.ones(npad, np.float64) if chain.scale is None else np.pad(chain.scale[l], (0, npad - chain.c_out[l])).astype(np.float64)
        y = _fma32(acc, sc, sh.astype(np.float64))
        last = l == L - 1
        if not (last and chain.linear) or mutant == "relu_on_linear":
            y = np.maximum(y, f(0))
        a = y if last else tf32_rn(y)
    C = chain.c_out[-1]
    if kind == "sa":
        b, npoint, ns = inp["idx"].shape
        g = a.reshape(b * npoint, ns, -1)
        out = g.max(1)
        if mutant == "pool_neighbour_sample":
            out = np.maximum(out, np.roll(g[:, 0], -1, 0))
        if mutant == "carry_leak" and ns > 64:
            first = g[:, :64].max(1)              # what a centre's first tile leaves in the carry
            out[1:] = np.maximum(out[1:], first[:-1])
        return np.ascontiguousarray(out[:, :C].reshape(b, npoint, C).transpose(0, 2, 1))
    if kind == "fp":
        b, n, _ = inp["idx"].shape
        return np.ascontiguousarray(a[:, :C].reshape(b, n, C).transpose(0, 2, 1))
    return a


# ------------------------------------------------------------------------------------------------ the case matrix
# name, kind, shape, chain (c_out, folded, linear), the kernel build each run takes (resident on / off).  The builds:
# resident <1,5> (widest layer 32), resident <4,4> (48..128), streaming <2,2> (<= 128), <4,1> (160..256), <8,1> (288..512);
# a warpgroup of the streaming kernel owns ceil(np/64) / floor(np/64) of the np/32 subtiles.
CASES = [
    # --- SA: b, n, npoint, ns, c_feat; out_stride_c extra channels and out_c_off
    dict(name="sa_f0_ns4_32", kind="sa", b=2, n=200, npoint=33, ns=4, c_feat=0, c_out=[32], folded=True, linear=False,
         extra=8, off=5, build="res<1,5> / <2,2>"),
    dict(name="sa_f1_ns8_16_32", kind="sa", b=2, n=300, npoint=70, ns=8, c_feat=1, c_out=[16, 32], folded=False, linear=False,
         extra=0, off=0, build="res<1,5> / <2,2>"),
    dict(name="sa_f2_ns16_48_64_lin", kind="sa", b=2, n=400, npoint=50, ns=16, c_feat=2, c_out=[48, 64], folded=False,
         linear=True, extra=36, off=20, build="res<4,4> / <2,2>"),
    dict(name="sa_f3_ns32_64_96_128", kind="sa", b=2, n=500, npoint=40, ns=32, c_feat=3, c_out=[64, 96, 128], folded=True,
         linear=False, extra=0, off=0, build="res<4,4> / <2,2>"),
    dict(name="sa_f4_ns64_32_32_lin", kind="sa", b=3, n=300, npoint=21, ns=64, c_feat=4, c_out=[32, 32], folded=False,
         linear=True, extra=3, off=3, build="res<1,5> / <2,2>"),
    dict(name="sa_f5_ns128_64_128", kind="sa", b=2, n=400, npoint=19, ns=128, c_feat=5, c_out=[64, 128], folded=True,
         linear=False, extra=0, off=0, build="res<4,4> / <2,2>"),
    dict(name="sa_f6_ns16_160", kind="sa", b=2, n=300, npoint=60, ns=16, c_feat=6, c_out=[160], folded=False, linear=False,
         extra=0, off=0, build="<4,1>"),
    dict(name="sa_f7_ns32_96_200", kind="sa", b=2, n=300, npoint=30, ns=32, c_feat=7, c_out=[96, 200], folded=True,
         linear=False, extra=10, off=4, build="<4,1>"),
    dict(name="sa_f8_ns8_288_lin", kind="sa", b=2, n=300, npoint=40, ns=8, c_feat=8, c_out=[288], folded=False, linear=True,
         extra=0, off=0, build="<8,1>"),
    dict(name="sa_f40_ns32_64_352", kind="sa", b=2, n=300, npoint=24, ns=32, c_feat=40, c_out=[64, 352], folded=True,
         linear=False, extra=0, off=0, build="<8,1>"),
    dict(name="sa_f96_ns64_128_416", kind="sa", b=2, n=200, npoint=12, ns=64, c_feat=96, c_out=[128, 416], folded=False,
         linear=False, extra=0, off=0, build="<8,1>"),
    dict(name="sa_f3_np1_ns128_480", kind="sa", b=3, n=200, npoint=1, ns=128, c_feat=3, c_out=[480], folded=True, linear=False,
         extra=0, off=0, build="<8,1>"),
    dict(name="sa_f1_ns32_32_512", kind="sa", b=2, n=300, npoint=16, ns=32, c_feat=1, c_out=[32, 512], folded=False,
         linear=False, extra=0, off=0, build="<8,1>"),
    dict(name="sa_f512_ns16_split3", kind="sa", b=2, n=64, npoint=8, ns=16, c_feat=512, c_out=[256, 384, 512], folded=False,
         linear=False, extra=64, off=32, build="<8,1> x3"),
    # --- FP: b, n, m, c_known, c_skip
    dict(name="fp_k3_s0_m3_32", kind="fp", b=2, n=100, m=3, c_known=3, c_skip=0, c_out=[32], folded=True, linear=False,
         build="res<1,5> / <2,2>"),
    dict(name="fp_k64_s1_64_48_lin", kind="fp", b=3, n=333, m=50, c_known=64, c_skip=1, c_out=[64, 48], folded=False,
         linear=True, build="res<4,4> / <2,2>"),
    dict(name="fp_k70_s5_96_128", kind="fp", b=2, n=999, m=300, c_known=70, c_skip=5, c_out=[96, 128], folded=False,
         linear=False, build="res<4,4> / <2,2>"),
    dict(name="fp_k256_s33_256_160", kind="fp", b=2, n=500, m=128, c_known=256, c_skip=33, c_out=[256, 160], folded=True,
         linear=False, build="<4,1>"),
    dict(name="fp_k64_s96_480_lin", kind="fp", b=2, n=300, m=64, c_known=64, c_skip=96, c_out=[480], folded=False, linear=True,
         build="<8,1>"),
    dict(name="fp_k256_s0_split2", kind="fp", b=2, n=130, m=40, c_known=256, c_skip=0, c_out=[512, 512], folded=False,
         linear=False, build="<8,1> x2"),
    # --- rows (prb_mlp_rows when the segment is a whole contiguous tensor, else prb_mlp_rows2): rows, c_a on a_pitch at
    # a_off, optional c_b on b_pitch at b_off (an offset that is not a multiple of 4 misaligns the base)
    dict(name="rows_1x1_32_lin", kind="rows", rows=1, c_a=1, c_out=[32], folded=False, linear=True, build="res<1,5> / <2,2>"),
    dict(name="rows_63x3_48", kind="rows", rows=63, c_a=3, c_out=[48], folded=True, linear=False, build="res<4,4> / <2,2>"),
    dict(name="rows_64x4_160", kind="rows", rows=64, c_a=4, c_out=[160], folded=False, linear=False, build="<4,1>"),
    dict(name="rows_65x5_64_224_lin", kind="rows", rows=65, c_a=5, c_out=[64, 224], folded=True, linear=True, build="<4,1>"),
    dict(name="rows_4097x31_32x3_lin", kind="rows", rows=4097, c_a=31, c_out=[32, 32, 32], folded=False, linear=True,
         build="res<1,5> / <2,2>"),
    dict(name="rows_1000x32_96", kind="rows", rows=1000, c_a=32, c_out=[96], folded=True, linear=False,
         build="res<4,4> / <2,2>"),
    dict(name="rows_700x33_288", kind="rows", rows=700, c_a=33, c_out=[288], folded=False, linear=False, build="<8,1>"),
    dict(name="rows_3000x99_64_96_128", kind="rows", rows=3000, c_a=99, c_out=[64, 96, 128], folded=True, linear=False,
         build="res<4,4> / <2,2>"),
    dict(name="rows_2000x259_128_196_256", kind="rows", rows=2000, c_a=259, c_out=[128, 196, 256], folded=False,
         linear=False, build="<4,1>"),
    dict(name="rows_1500x515_split3_lin", kind="rows", rows=1500, c_a=515, c_out=[256, 384, 512], folded=True, linear=True,
         build="<8,1> x3"),
    dict(name="rows_700x1536_split2", kind="rows", rows=700, c_a=1536, c_out=[512, 512], folded=False, linear=False,
         build="<8,1> x2"),
    dict(name="rows_2000x256_128_image_lin", kind="rows", rows=2000, c_a=256, c_out=[128], folded=False, linear=True,
         build="<2,2> (image over half of shared memory)"),
    dict(name="rows2_a5p8", kind="rows", rows=500, c_a=5, a_pitch=8, a_off=0, c_out=[64], folded=True, linear=False,
         build="res<4,4> / <2,2>"),
    dict(name="rows2_a6p12_b33p40_lin", kind="rows", rows=777, c_a=6, a_pitch=12, a_off=0, c_b=33, b_pitch=40, b_off=4,
         c_out=[96, 32], folded=False, linear=True, build="res<4,4> / <2,2>"),
    dict(name="rows2_misaligned", kind="rows", rows=300, c_a=33, a_pitch=45, a_off=1, c_b=7, b_pitch=45, b_off=35,
         c_out=[48], folded=True, linear=False, build="res<4,4> / <2,2>"),
    dict(name="rows2_a128p132_b5p16", kind="rows", rows=1000, c_a=128, a_pitch=132, a_off=0, c_b=5, b_pitch=16, b_off=4,
         c_out=[128], folded=False, linear=False, build="res<4,4> / <2,2>"),
]
BY_NAME = {c["name"]: c for c in CASES}

# many-tile cases: run under these prb_options as well, so one CTA walks hundreds of items
PERSIST_CASES = [
    dict(name="sa_persist_f1_ns32_16_16_32", kind="sa", b=2, n=2048, npoint=1024, ns=32, c_feat=1, c_out=[16, 16, 32],
         folded=True, linear=False, extra=0, off=0, build="res<1,5> / <2,2>"),
    dict(name="rows_persist_20000x99_64_288", kind="rows", rows=20000, c_a=99, c_out=[64, 288], folded=False, linear=False,
         build="<8,1>"),
]
PERSIST_OPTIONS = [dict(mlp_sms=1), dict(mlp_sms=1, mlp_occ=1)]


def pack_args(case):
    """(kind, split, c_in) the chain of a case is packed with"""
    if case["kind"] == "sa":
        return 0, case["c_feat"], 3 + case["c_feat"]
    if case["kind"] == "fp":
        return 1, case["c_known"], case["c_known"] + case["c_skip"]
    c_b = case.get("c_b", 0)
    return (1, case["c_a"], case["c_a"] + c_b) if c_b else (2, 0, case["c_a"])


def reduced(case):
    """the same channels at a size an fp32 emulation runs in a moment (two or more centres / scenes kept)"""
    c = dict(case)
    if c["kind"] == "sa":
        c["b"] = min(c["b"], 2)
        c["npoint"] = min(c["npoint"], max(2, 256 // c["ns"]))
    elif c["kind"] == "fp":
        c["b"], c["n"] = min(c["b"], 2), min(c["n"], 70)
    else:
        c["rows"] = min(c["rows"], 130)
    return c


def make(case, seed=0):
    """(chain, packed image, unpacked layers, host inputs) of a case"""
    rng = np.random.default_rng([seed] + [ord(ch) for ch in case["name"]])
    kind, split, c_in = pack_args(case)
    chain = Chain(rng, kind, split, c_in, case["c_out"], case["folded"], case["linear"])
    img, layers = chain.packed()
    if case["kind"] == "sa":
        inp = sa_inputs(rng, case["b"], case["n"], case["npoint"], case["ns"], case["c_feat"])
    elif case["kind"] == "fp":
        inp = fp_inputs(rng, case["b"], case["n"], case["m"], case["c_known"], case["c_skip"])
    else:
        inp = rows_inputs(rng, case["rows"], case["c_a"], case.get("a_pitch", case["c_a"]), case.get("a_off", 0),
                          case.get("c_b", 0), case.get("b_pitch", 0), case.get("b_off", 0))
    return chain, img, layers, inp
