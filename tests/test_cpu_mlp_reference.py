"""The float64 reference of the MLP chain (mlp_reference.py) checked on the host: its weight unpacker against the packer,
its error bound against an fp32 model of the kernel, and its power to catch subtle mistakes planted in that model."""
import numpy as np
import pytest

import mlp_reference as R
from pointrcnn_b200 import mlp_chain

# --------------------------------------------------------------------------------------------- unpacker
PACK_CASES = sorted({(R.pack_args(c), tuple(c["c_out"])) for c in R.CASES + R.PERSIST_CASES})
PACK_CASES += [((0, f, 3 + f), (31, 33)) for f in range(9)]                # SA: every c_feat up to the separate segment
PACK_CASES += [((1, 33, 40), (1, 196)), ((1, 64, 64), (48,))]              # FP: two segments, and no skip segment
PACK_CASES += [((2, 0, 7), (1, 31, 33)), ((2, 0, 300), (196, 512, 1))]     # every width


@pytest.mark.parametrize("args,c_out", PACK_CASES, ids=["kind%d_split%d_cin%d_" % a + "_".join(map(str, c)) for a, c in PACK_CASES])
def test_unpack_inverts_the_packer(args, c_out):
    """unpack(prb_mlp_pack_weights_ex(W)) is tf32_rna(W), bit for bit, with zero padding"""
    kind, split, c_in = args
    rng = np.random.default_rng(c_in * 7 + len(c_out))
    dims = [c_in] + list(c_out)
    ws = [rng.standard_normal((co, ci)).astype(np.float32) for ci, co in zip(dims[:-1], dims[1:])]
    img = mlp_chain.pack_image(kind, split, ws)
    layers = R.unpack(img, kind, split, c_in, list(c_out))
    for W, ly in zip(ws, layers):
        assert ly.W.shape == W.shape
        assert np.array_equal(ly.W.view(np.uint32), R.tf32_rna(W).view(np.uint32))


def test_unpack_rejects_a_wrong_layout():
    """the unpacker does not just mirror the packer: an image with a unit swizzled the wrong way is refused or differs"""
    rng = np.random.default_rng(1)
    W = rng.standard_normal((40, 37)).astype(np.float32)
    img = mlp_chain.pack_image(2, 0, [W])
    bad = img.copy()
    bad[4:8], bad[8:12] = img[8:12], img[4:8]          # row 0, units 1 and 2 of the first chunk swapped
    assert np.array_equal(R.unpack(img, 2, 0, 37, [40])[0].W, R.tf32_rna(W))
    assert not np.array_equal(R.unpack(bad, 2, 0, 37, [40])[0].W, R.tf32_rna(W))
    with pytest.raises(AssertionError):
        R.unpack(img[:-32], 2, 0, 37, [40])


# --------------------------------------------------------------------------------------------- soundness
ALL = R.CASES + R.PERSIST_CASES


@pytest.mark.parametrize("case", ALL, ids=[c["name"] for c in ALL])
def test_bound_holds_for_fp32_accumulation_orders(case):
    """an fp32 model of the kernel (its rounding points, fp32 accumulation per K chunk) sits inside the bound for every
    case shape, whichever order the products of a chunk are added in"""
    c = R.reduced(case)
    chain, img, layers, inp = R.make(c)
    ref, bound = R.expected(c["kind"], chain, layers, inp)
    worst = 0.0
    for order in R.ORDERS:
        got = R.emulate(c["kind"], chain, layers, inp, order)
        assert got.shape == ref.shape and np.isfinite(got).all()
        ok, ratio, bad = R.check(got, ref, bound)
        assert ok, "%s, %s order: %d elements outside the bound, max err/bound %.3g" % (c["name"], order, bad, ratio)
        worst = max(worst, ratio)
    assert worst > 0, "the emulation matched the float64 reference exactly: the bound was not exercised"


# --------------------------------------------------------------------------------------------- sensitivity
# each planted mistake, and a case of the matrix whose check must catch it
MUTANT_CASES = {
    "drop_partial_kstep": "sa_f40_ns32_64_352",        # layer 0 chunks of 4, 1 and 1 K-steps
    "shift_off_by_one": "rows_1000x32_96",
    "skip_transposed": "fp_k70_s5_96_128",
    "fp_weights_swapped": "fp_k70_s5_96_128",
    "rel_xyz_next_centre": "sa_f3_ns32_64_96_128",
    "pool_neighbour_sample": "sa_f2_ns16_48_64_lin",
    "carry_leak": "sa_f5_ns128_64_128",                # two tiles per centre
    "relu_on_linear": "rows_4097x31_32x3_lin",
}


def test_every_mutant_has_a_case():
    assert sorted(MUTANT_CASES) == sorted(R.MUTANTS)


@pytest.mark.parametrize("mutant", R.MUTANTS)
def test_bound_catches_a_subtly_wrong_kernel(mutant):
    c = R.reduced(R.BY_NAME[MUTANT_CASES[mutant]])
    chain, img, layers, inp = R.make(c)
    ref, bound = R.expected(c["kind"], chain, layers, inp)
    assert R.check(R.emulate(c["kind"], chain, layers, inp), ref, bound)[0], "the unmutated model must pass"
    ok, ratio, bad = R.check(R.emulate(c["kind"], chain, layers, inp, mutant=mutant), ref, bound)
    assert not ok, "mutant %s passed the check on %s" % (mutant, c["name"])
    print("mutant %-22s caught on %-24s: %d elements outside the bound, max err/bound %.3g" % (mutant, c["name"], bad, ratio))
