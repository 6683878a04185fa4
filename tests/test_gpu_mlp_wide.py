"""The wide-layer kernel: every chain layer wider than 256 runs alone on mlp_wide_kernel, over rows in global memory, as
128-row x 256-column tiles (two 64-row warpgroups, one m64n256k8 per K=8 step).  A wide first layer reads its operand
from rows the gather kernel wrote (tf32, padded segment order); a wide later layer reads the rows the launch before it
wrote.

Every case is checked element by element against the float64 reference and error bound of mlp_reference.py.  The
cases: every wide launch of the RPN backbone forward at B = 16 and the RCNN stage's SA3 chain; row counts that leave a
partial or empty second warpgroup in the last 128-row block; SA centres of 4 .. 128 samples pooled from a wide last
layer; K tails (layer-0 widths that are not multiples of 32); FP with and without skip and point-major copy; a linear
last layer; 1-3 layer chains whose wide layer is first, middle or last; 384- and 288-wide layers whose last column block
is narrower than 256; an FP3 module at B = 16 whose projection of the known points and main chain both run wide.

The last two tests simulate, on the host, the two mistakes a 128-row x two-column-block tile invites -- the second
warpgroup computing from the first one's A rows, and the second column block reading the first block's weights --
and show that the float64 check rejects the outputs such a kernel would give.  They plant nothing in the kernel: the
check's power to catch a kernel with either mistake rests on it rejecting these outputs.
"""
import ctypes

import numpy as np
import pytest
import torch

import mlp_reference as R
import module_reference as MR
from test_gpu_mlp_reference import SENTINEL, Launch
from test_gpu_module_reference import check_fp

pytestmark = pytest.mark.gpu

from pointrcnn_b200 import _cabi as C  # noqa: E402
from pointrcnn_b200 import config  # noqa: E402
from pointrcnn_b200.pointnet2 import pointnet2_modules as pm  # noqa: E402


def _sa(name, b, n, npoint, ns, c_feat, c_out, folded=True, linear=False, extra=0, off=0):
    return dict(name=name, kind="sa", b=b, n=n, npoint=npoint, ns=ns, c_feat=c_feat, c_out=c_out, folded=folded,
                linear=linear, extra=extra, off=off, build="wide")


def _fp(name, b, n, m, c_known, c_skip, c_out, folded=True, linear=False):
    return dict(name=name, kind="fp", b=b, n=n, m=m, c_known=c_known, c_skip=c_skip, c_out=c_out, folded=folded,
                linear=linear, build="wide")


def _rows(name, rows, c_a, c_out, folded=True, linear=False, **kw):
    return dict(name=name, kind="rows", rows=rows, c_a=c_a, c_out=c_out, folded=folded, linear=linear, build="wide", **kw)


# the chains of the RPN backbone forward at B = 16 x 16384 points with a layer wider than 256 (SA4's two radii into one
# 1024-channel output, FP3, FP2), and the RCNN stage's SA3 chain (all 32 points of a RoI's SA2 output in one centre)
RPN_CASES = [
    _sa("rpn_sa4_ns16", 16, 256, 64, 16, 512, [256, 256, 512], extra=512, off=0),
    _sa("rpn_sa4_ns32", 16, 256, 64, 32, 512, [256, 384, 512], extra=512, off=512),
    _fp("rpn_fp3", 16, 256, 64, 1024, 512, [512, 512]),
    _fp("rpn_fp2", 16, 1024, 256, 512, 256, [512, 512]),
    _sa("rcnn_sa3", 100, 32, 1, 32, 256, [256, 256, 512]),
]

CASES = [
    # row counts against 128-row blocks: one row; 100 (the second warpgroup partial); 128 + 1 (the last block's second
    # warpgroup empty); 200 (its second warpgroup partial); K tails of 515 and 259 inputs
    _rows("rows_1x515_512", 1, 515, [512]),
    _rows("rows_100x259_384_lin", 100, 259, [384], linear=True),
    _rows("rows_129x515_512", 129, 515, [512], folded=False),
    _rows("rows_200x259_288", 200, 259, [288]),
    _rows("rows2_333x5p8_b19p24_320", 333, 5, [320], a_pitch=8, a_off=0, c_b=19, b_pitch=24, b_off=4, folded=False),
    # the wide layer first, in the middle, last; two wide layers in a row
    _rows("rows_300x70_512_96", 300, 70, [512, 96]),
    _rows("rows_257x33_64_416_64_lin", 257, 33, [64, 416, 64], linear=True),
    _rows("rows_130x40_96_128_300", 130, 40, [96, 128, 300], folded=False),
    _rows("rows_400x64_384_512_lin", 400, 64, [384, 512], linear=True),
    # SA: every centre size from a wide last layer; a wide first layer over the gathered rows
    _sa("sa_ns4_f0_288", 2, 300, 35, 4, 0, [288], folded=False),
    _sa("sa_ns8_f1_64_512_lin", 2, 400, 41, 8, 1, [64, 512], linear=True, extra=7, off=3),
    _sa("sa_ns16_f13_512_196_256", 2, 200, 17, 16, 13, [512, 196, 256]),
    _sa("sa_ns32_f64_256_384", 2, 400, 21, 32, 64, [256, 384], folded=False),
    _sa("sa_ns64_f20_96_512", 2, 300, 13, 64, 20, [96, 512]),
    _sa("sa_ns128_f5_128_512", 2, 400, 19, 128, 5, [128, 512]),
    _sa("sa_ns128_f40_320_lin", 2, 300, 9, 128, 40, [320], folded=False, linear=True),
    # FP: with and without skip, K tails in both segments, a wide layer after a narrow one
    _fp("fp_k64_s0_512", 2, 333, 50, 64, 0, [512]),
    _fp("fp_k70_s5_352_128_lin", 2, 999, 300, 70, 5, [352, 128], folded=False, linear=True),
    _fp("fp_k129_s33_160_512", 3, 257, 64, 129, 33, [160, 512], folded=False),
    _fp("fp_k64_s16_512_256_256", 2, 130, 40, 64, 16, [512, 256, 256], folded=False),
]


def _run(case, cuda):
    chain, _, layers, inp = R.make(case)
    ref, bound = R.expected(case["kind"], chain, layers, inp)
    launch = Launch(case, chain, inp, cuda)
    launch.verify(launch.run(), ref, bound, case["name"])
    return launch


@pytest.mark.parametrize("case", RPN_CASES + CASES, ids=[c["name"] for c in RPN_CASES + CASES])
def test_wide(cuda, case):
    _run(case, cuda)


@pytest.mark.parametrize("name", ["fp_k64_s0_512", "fp_k129_s33_160_512", "rpn_fp2"])
def test_wide_fp_without_point_major(cuda, name):
    """without out_pm the channel-major output keeps the same bits"""
    case = next(c for c in RPN_CASES + CASES if c["name"] == name)
    launch = _run(case, cuda)
    I, (flat, out) = launch.inp, launch.bufs[0]
    with_pm = launch.run()[0]
    flat.fill_(SENTINEL)
    C.check(launch.lib.prb_fp_interp_mlp_ws(case["b"], case["n"], case["m"], case["c_known"], case["c_skip"],
                                            C.ptr(I["known_pm"]), C.ptr(I["idx"]), C.ptr(I["weight"]),
                                            C.ptr(I["skip"]) if case["c_skip"] else None, ctypes.byref(launch.desc),
                                            C.ptr(out), None, C.ptr(launch.ws), C.c_size_t(launch.wsb), C.stream()),
            case["name"])
    torch.cuda.synchronize()
    np.testing.assert_array_equal(flat.cpu().numpy().view(np.int32), with_pm.view(np.int32))


def test_wide_after_fp3_projection(cuda):
    """FP3 at B = 16 with the known points projected (fp_project_min_rows lowered to admit it): the projection, a linear
    1024 -> 512 rows chain, and the main chain [interp 512 | skip 512] -> 512, 512 both run on the wide kernel"""
    torch.manual_seed(0)
    fp = MR.seeded(pm.PointnetFPModule(mlp=[1024 + 512, 512, 512]), 11).to(cuda).eval()
    b, n, m = 16, 256, 64
    unknown = torch.rand(b, n, 3, device=cuda) * 40.0
    known = unknown[:, torch.randperm(n, device=cuda)[:m]].contiguous()
    skip = torch.randn(b, 512, n, device=cuda)
    known_feats = torch.randn(b, 1024, m, device=cuda)
    with torch.no_grad(), config.override(fp_project_min_rows=0):
        out = fp(unknown, known, skip, known_feats)
        assert check_fp(fp, unknown, known, skip, known_feats, out, "FP3 projected, B = 16"), "FP3 was not projected"


def test_wide_header_form_refuses_without_workspace(cuda):
    """the SA entry without a workspace cannot materialise the rows a wide layer reads: it refuses, and writes nothing"""
    case = RPN_CASES[0]
    chain, _, layers, inp = R.make(dict(case, b=1))
    launch = Launch(dict(case, b=1), chain, inp, cuda)
    I, (flat, out) = launch.inp, launch.bufs[0]
    flat.fill_(SENTINEL)
    rc = launch.lib.prb_sa_group_mlp_max(1, case["n"], case["npoint"], case["ns"], case["c_feat"], C.ptr(I["xyz"]),
                                         C.ptr(I["new_xyz"]), C.ptr(I["feats_pm"]), C.ptr(I["idx"]),
                                         ctypes.byref(launch.desc), C.ptr(out), launch.stride, 0, C.stream())
    torch.cuda.synchronize()
    assert rc != 0
    assert (flat.cpu().numpy() == SENTINEL).all()


# ------------------------------------------------------------------------------------------------ planted mistakes
def _rows_output(cuda, name):
    case = next(c for c in CASES if c["name"] == name)
    chain, _, layers, inp = R.make(case)
    ref, bound = R.expected(case["kind"], chain, layers, inp)
    launch = Launch(case, chain, inp, cuda)
    flat = launch.run()[0]
    got = flat[:case["rows"] * launch.pitch].reshape(case["rows"], launch.pitch)[:, :chain.c_out[-1]]
    return chain, layers, inp, got.copy(), ref[:, :chain.c_out[-1]], bound[:, :chain.c_out[-1]]


def _caught(label, got, ref, bound):
    ok, ratio, bad = R.check(got, ref, bound)
    print("%s: caught by the float64 bound check, %d elements outside, max err/bound %.3g" % (label, bad, ratio))
    return not ok


def test_wide_catches_second_warpgroup_reading_first_rows(cuda):
    """simulated: rows 64-127 of each 128-row block computed from rows 0-63 repeat the first half's output"""
    chain, layers, inp, got, ref, bound = _rows_output(cuda, "rows_129x515_512")
    assert R.check(got, ref, bound)[0]
    bad = got.copy()
    bad[64:128] = got[0:64]
    assert _caught("second warpgroup reads the first one's A rows", bad, ref, bound)


def test_wide_catches_dropped_column_block_offset(cuda):
    """simulated: in both wide layers (384 = 2 x 192 and 512 = 2 x 256 columns) the second column block multiplies the
    first block's weight rows, and the 384-wide layer's wrong columns reach every column of the 512-wide one"""
    chain, layers, inp, got, ref, bound = _rows_output(cuda, "rows_400x64_384_512_lin")
    assert R.check(got, ref, bound)[0]
    a, e = R.layer0("rows", inp)
    mutated = []
    for ly in layers:
        W = ly.W.copy()
        bw = 32 * ((R.round_up(W.shape[0], 32) // 32 + 1) // 2)    # the kernel's column block width
        W[bw:] = W[:W.shape[0] - bw]
        mutated.append(R.Layer(W, ly.Wk, ly.kmap))
    bad = R.reference(chain, mutated, a, e)[0][:, :chain.c_out[-1]].astype(np.float32)
    assert _caught("column block offset dropped from the B slab", bad, ref, bound)
