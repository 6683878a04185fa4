"""The float64 FP training reference (tests/fp_train_reference.py) on the CPU: its two layer-0 orders agree, it agrees
with the torch module, the planted mistakes fail its tolerances, and the integer cases meet their exactness
preconditions."""
import pytest
import torch

import fp_train_reference as R


def _case(B=2, n=96, m=24, ci=12, cs=5, widths=(16, 8), bn=True, seed=0):
    g = torch.Generator().manual_seed(seed)
    known = torch.randn(B, ci, m, generator=g)
    skip = torch.randn(B, cs, n, generator=g) if cs else None
    idx = torch.stack([torch.stack([torch.randperm(m, generator=g)[:3] for _ in range(n)]) for _ in range(B)]).int()
    w = torch.rand(B, n, 3, generator=g) + 0.1
    w = w / w.sum(2, keepdim=True)
    layers, c_in = [], ci + cs
    for co in widths:
        L = dict(W=torch.randn(co, c_in, generator=g) / c_in ** 0.5)
        if bn:
            L.update(gamma=1 + 0.1 * torch.randn(co, generator=g), beta=0.1 * torch.randn(co, generator=g))
        else:
            L["bias"] = 0.1 * torch.randn(co, generator=g)
        layers.append(L)
        c_in = co
    gout = torch.randn(B, widths[-1], n, generator=g)
    return known, skip, idx, w, layers, gout


def _run(case, bn, order="plain", mutant=None):
    known, skip, idx, w, layers, gout = case
    out, cache = R.forward(known, skip, idx, w, layers, bn, order=order, mutant=mutant)
    return out, R.backward(cache, gout)


def _all_ok(a, b):
    oa, ga = a
    ob, gb = b
    checks = [R.compare(oa, ob, "fwd")]
    for k in ("W", "gamma", "beta", "bias"):
        for x, y in zip(ga[k], gb[k]):
            if x is not None:
                checks.append(R.compare(x, y, "grad"))
    checks.append(R.compare(ga["known"], gb["known"], "grad"))
    if ga.get("skip") is not None and ga["skip"].numel():
        checks.append(R.compare(ga["skip"], gb["skip"], "grad"))
    return all(ok for ok, _ in checks)


@pytest.mark.parametrize("bn", [True, False])
def test_plain_and_projected_orders_agree(bn):
    case = _case(bn=bn)
    a, b = _run(case, bn, "plain"), _run(case, bn, "projected")
    assert torch.allclose(a[0], b[0], atol=1e-12)
    for x, y in zip(a[1]["W"], b[1]["W"]):
        assert torch.allclose(x, y, atol=1e-10)
    assert torch.allclose(a[1]["known"], b[1]["known"], atol=1e-10)
    assert torch.allclose(a[1]["skip"], b[1]["skip"], atol=1e-10)


@pytest.mark.parametrize("bn", [True, False])
def test_reference_matches_the_torch_module(bn):
    from pointrcnn_b200.pointnet2 import pytorch_utils as pt_utils
    known, skip, idx, w, layers, gout = case = _case(bn=bn)
    mlp = pt_utils.SharedMLP([known.size(1) + skip.size(1)] + [L["W"].shape[0] for L in layers], bn=bn).double().train()
    with torch.no_grad():
        for layer, L in zip(mlp.children(), layers):
            layer.conv.weight.copy_(L["W"].view_as(layer.conv.weight))
            if bn:
                layer.bn.bn.weight.copy_(L["gamma"])
                layer.bn.bn.bias.copy_(L["beta"])
            else:
                layer.conv.bias.copy_(L["bias"])
    kf = known.double().requires_grad_(True)
    sk = skip.double().requires_grad_(True)
    interp = R._interp(kf.transpose(1, 2), idx, w.double()).transpose(1, 2)
    out = mlp(torch.cat([interp, sk], 1).unsqueeze(-1)).squeeze(-1)
    out.backward(gout.double())
    ref_out, ref = _run(case, bn)
    assert torch.allclose(out, ref_out, atol=1e-10)
    assert torch.allclose(kf.grad, ref["known"], atol=1e-10)
    assert torch.allclose(sk.grad, ref["skip"], atol=1e-10)
    for layer, gw in zip(mlp.children(), ref["W"]):
        assert torch.allclose(layer.conv.weight.grad.view_as(gw), gw, atol=1e-10)


@pytest.mark.parametrize("mutant", R.MUTANTS)
@pytest.mark.parametrize("order", ["plain", "projected"])
def test_planted_mistakes_fail_the_tolerances(mutant, order):
    case = _case(bn=True, seed=3)
    good = _run(case, True, order)
    bad = _run(case, True, order, mutant)
    assert not _all_ok(good, bad), mutant


def test_the_tolerances_accept_the_other_order():
    case = _case(seed=4)
    assert _all_ok(_run(case, True, "plain"), _run(case, True, "projected"))


@pytest.mark.parametrize("taps,widths", [("half", (16,)), ("onehot", (16, 8, 4)), ("onehot", (128, 128))])
def test_integer_cases_meet_the_exactness_preconditions(taps, widths):
    c = R.integer_case(2, 64, 16, 12, 3, widths, seed=1, taps=taps)
    out, cache = R.forward(c["known"], c["skip"], c["idx"], c["w"], c["layers"], False)
    grads = R.backward(cache, c["gout"])
    R.check_exact(c, cache, out, grads)


def test_the_exactness_check_rejects_an_inexact_operand():
    c = R.integer_case(1, 32, 8, 4, 2, (8,), seed=2)
    c["known"][0, 0, 0] = 1.0 / 3.0
    out, cache = R.forward(c["known"], c["skip"], c["idx"], c["w"], c["layers"], False)
    with pytest.raises(AssertionError):
        R.check_exact(c, cache, out, R.backward(cache, c["gout"]))
