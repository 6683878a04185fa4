"""The per-element bound of tests/train_bound.py against an fp32 emulation of the SA and FP training kernels, without a GPU:
every element of every output, running statistic and gradient stays inside its bound under several accumulation orders,
and each planted mistake (train_bound.SA_MUTANTS / FP_MUTANTS) is caught.  Each mutant prints its largest error / bound
under the per-element bound and under the old tensor-wide tolerances; OLD_MISSES records which the tensor-wide
tolerances let through, and the test keeps that record true."""
import pytest
import torch

import sa_train_reference as R
import train_bound as TB


def _bn_layers(g, widths, c_in):
    """BN layers (layer_params form, fp32-representable values): gammas in [0.5, 1.5] but channels 0 and 1 of every layer
    at 1e-3 and -2e-3, and layer 0's channel 3 has a zero weight row (a constant channel: zero variance)"""
    out = []
    for co in widths:
        w = (torch.randn(co, c_in, generator=g) * (2.0 / c_in) ** 0.5).float()
        ga = (torch.rand(co, generator=g) + 0.5).float()
        ga[0], ga[1] = 1e-3, -2e-3
        if not out:
            w[3] = 0
        out.append(dict(w=w.double(), b=None, gamma=ga.double(), beta=(torch.rand(co, generator=g) * 0.4 - 0.2).float().double(),
                        rm=torch.randn(co, generator=g).float().double(), rv=(torch.rand(co, generator=g) + 0.5).float().double(),
                        nbt=1, eps=1e-5, momentum=0.1))
        c_in = co
    return out


def sa_case(seed=0, B=2, N=96, npoint=8):
    """two scales (ns 8 and 16) over a cloud with duplicated points, the intensity channel offset by 16 so that layer 0's
    channels have |mean| >> std"""
    g = torch.Generator().manual_seed(seed)
    xyz = torch.rand(B, N, 3, generator=g)
    feats = torch.rand(B, 1, N, generator=g) + 16.0
    xyz[:, N - 8:] = xyz[:, :8]                         # duplicates: same coordinates and features, other indices
    feats[:, :, N - 8:] = feats[:, :, :8]
    cidx = torch.arange(npoint) * (N // npoint)
    centres = xyz[:, cidx].contiguous()
    scales = []
    for radius, ns, widths in ((0.3, 8, (16, 16, 32)), (0.6, 16, (32, 32, 64))):
        scales.append(dict(idx=R.ball_query(radius, ns, xyz, centres).int(), layers=_bn_layers(g, widths, 4)))
    C = sum(s["layers"][-1]["w"].shape[0] for s in scales)
    grad_out = torch.randn(B, C, npoint, generator=g)
    return dict(xyz=xyz, centres=centres, feats=feats, scales=scales, grad_out=grad_out)


def fp_case(seed=0, B=2, n=40, m=12, ci=6, cs=3):
    g = torch.Generator().manual_seed(seed)
    known = torch.randn(B, ci, m, generator=g)
    known[:, 0] += 30.0                                  # an offset input channel
    skip = torch.randn(B, cs, n, generator=g)
    idx = torch.stack([torch.stack([torch.randperm(m, generator=g)[:3] for _ in range(n)]) for _ in range(B)]).int()
    w = torch.rand(B, n, 3, generator=g) + 0.05
    w = (w / w.sum(-1, keepdim=True)).float()
    layers = _bn_layers(g, (16, 8), ci + cs)
    return dict(known=known, skip=skip, idx=idx, w=w, layers=layers, grad_out=torch.randn(B, 8, n, generator=g))


def _decisions(st):
    return st.flips


def run_sa(case, order, mutant=None):
    """the emulation and its replay -> (ratios under the bound, under the tensor-wide tolerances, decisions under the
    bound, decisions under the tensor-wide check)"""
    c = case
    gf = torch.zeros_like(c["feats"])
    new, old, dec_new, dec_old, parts, off, sts = {}, {}, 0.0, 0.0, [], 0, []
    for k, s in enumerate(c["scales"]):
        C = s["layers"][-1]["w"].shape[0]
        gout = c["grad_out"][:, off:off + C].contiguous()
        emu = TB.emulate_sa(c["xyz"], c["centres"], c["feats"], s["idx"], s["layers"], gout, order, mutant, grad_feats=gf)
        st = TB.sa_scale(c["xyz"], c["centres"], c["feats"], s["idx"], s["layers"], emu["z"], emu["stats"], emu["chosen"], gout)
        parts.append(st.feats)
        worst, not_first = st.pool
        dec_new = max(dec_new, _decisions(st), worst, float("inf") if not_first else 0.0)
        dec_old = max(dec_old, TB.old_pool_check(emu["chosen"], st, s["idx"].shape[2]))
        sts.append((emu, st))
        off += C
    fg = TB.feats_grad(parts)
    for k, (emu, st) in enumerate(sts):
        last = k == len(sts) - 1
        for q, r in TB.ratios(emu, st, (gf, fg) if last else None).items():
            new[q if q == "feats" else "s%d.%s" % (k, q)] = r
        for q, r in TB.old_ratios(emu, st, (gf, fg) if last else None).items():
            old[q if q == "feats" else "s%d.%s" % (k, q)] = r
    return new, old, dec_new, dec_old


def run_fp(case, order, mutant=None):
    c = case
    emu = TB.emulate_fp(c["known"], c["skip"], c["idx"], c["w"], c["layers"], c["grad_out"], order, mutant)
    st = TB.fp_module(c["known"], c["skip"], c["idx"], c["w"], c["layers"], emu["z"], emu["stats"], c["grad_out"])
    return TB.ratios(emu, st), TB.old_ratios(emu, st), _decisions(st), 0.0


RUN = {"sa": (sa_case, run_sa), "fp": (fp_case, run_fp)}


@pytest.mark.parametrize("order", TB.ORDERS)
@pytest.mark.parametrize("kind", ["sa", "fp"])
def test_the_fp32_emulation_stays_inside_the_bound(kind, order):
    make, run = RUN[kind]
    for seed in (0, 1):
        new, _, dec, _ = run(make(seed), order)
        worst = max(new, key=new.get)
        print("%s %s seed %d: worst error / bound %.3g (%s), decisions %.3g" % (kind, order, seed, new[worst], worst, dec))
        assert new[worst] <= 1.0, (worst, new)
        assert dec <= 1.0


# The mutants the tensor-wide tolerances (sa_train_reference.FWD_TOL / GRAD_TOL / FROB_TOL and the decision check of
# test_gpu_sa_train) let through on these cases.  A quantity counts as a catch only where the correct emulation passes
# the tolerance: with the intensity offset, the correct layer-0 weight gradient of the SA cases already fails it (its
# intensity column is a sum of 16 dZ that BN makes cancel, so the fp32 rounding of the summands dominates), so mistakes
# visible only there count as missed.
OLD_MISSES = {"sa": {"biased_running", "no_sum_gx_small_gamma", "drop_xyz_grad", "pool_last_max"}, "fp": set()}
_CLEAN = {}


@pytest.mark.parametrize("kind,mutant", [("sa", m) for m in TB.SA_MUTANTS] + [("fp", m) for m in TB.FP_MUTANTS])
def test_every_mutant_is_caught(kind, mutant):
    make, run = RUN[kind]
    if kind not in _CLEAN:
        _CLEAN[kind] = run(make(0), "sequential")
    _, clean_old, _, clean_dec_old = _CLEAN[kind]
    new, old, dec_new, dec_old = run(make(0), "sequential", mutant)
    worst = max(max(new.values()), dec_new)
    where = max(new, key=new.get) if max(new.values()) >= dec_new else "decisions"
    fair = {q: r for q, r in old.items() if clean_old[q] <= 1.0}
    worst_old = max(max(fair.values()), dec_old if clean_dec_old <= 1.0 else 0.0)
    print("%s %s: largest error / bound %.3g (%s); under the tensor-wide tolerances %.3g (%s; all quantities %.3g)"
          % (kind, mutant, worst, where, worst_old, max(fair, key=fair.get), max(old.values())))
    assert worst > 1.0, new
    assert (worst_old <= 1.0) == (mutant in OLD_MISSES[kind]), (mutant, worst_old, old)


def test_tf32_rounds_to_nearest_even():
    # the emulation's operand rounding is the kernels' cvt.rn.tf32: ties go to the even 10-bit mantissa
    x = torch.tensor([1.0 + 2 ** -11, 1.0 + 3 * 2 ** -11, -(1.0 + 2 ** -11), 1.0 + 2 ** -11 + 2 ** -20, float("inf")])
    want = torch.tensor([1.0, 1.0 + 2 ** -9, -1.0, 1.0 + 2 ** -10, float("inf")])
    assert torch.equal(TB.tf32(x), want)


def test_weight_gradient_split_matches_the_kernel_rule():
    # st_wsplit: about 528 CTAs, chunks a multiple of 32 rows; RPN SA1 scale 0 layer 0 (4 -> 16) at B = 16
    assert TB.wsplit(16 * 4096 * 16, 16, 4) == (2016, 521)
    assert TB.wsplit(100, 16, 4) == (128, 1)
