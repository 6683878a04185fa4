"""The streaming chain kernel's tile pair: launches whose widest layer is 129-256 wide (and whose pair fits a three-stage
weight ring) run tiles 2u and 2u + 1 in one CTA, each weight chunk streamed once for both.

Where the resident kernel also runs a chain (every layer at most 128 wide, image at most half of shared memory), the
two kernels must agree bit for bit: prb_options.mlp_resident = 1 against 0, compared as int32 bit patterns.  Every case is
also checked element by element against the float64 reference and error bound of mlp_reference.py, which is the only
check for chains 129-256 wide.  The cases: every RPN launch at B = 16 up to 256 wide that streams (SA3 pairs, FP1 and
FP0 single tiles); odd tile counts and partial last tiles; 4 .. 128 samples per SA centre; FP with and without skip, with
and without the point-major copy; chains whose last segment runs from materialised rows; 1-3 layers and K tails.
"""
import ctypes

import numpy as np
import pytest
import torch

import mlp_reference as R
from test_gpu_mlp_reference import SENTINEL, Launch

pytestmark = pytest.mark.gpu

from pointrcnn_b200 import _cabi as C  # noqa: E402


def _sa(name, b, n, npoint, ns, c_feat, c_out, folded=True, linear=False, extra=0, off=0):
    return dict(name=name, kind="sa", b=b, n=n, npoint=npoint, ns=ns, c_feat=c_feat, c_out=c_out, folded=folded,
                linear=linear, extra=extra, off=off, build="pair")


def _fp(name, b, n, m, c_known, c_skip, c_out, folded=True, linear=False):
    return dict(name=name, kind="fp", b=b, n=n, m=m, c_known=c_known, c_skip=c_skip, c_out=c_out, folded=folded,
                linear=linear, build="pair")


def _rows(name, rows, c_a, c_out, folded=True, linear=False, **kw):
    return dict(name=name, kind="rows", rows=rows, c_a=c_a, c_out=c_out, folded=folded, linear=linear, build="pair", **kw)


# the streamed launches up to 256 wide of the RPN backbone forward at B = 16 x 16384 points: SA3 (two radii, 512 output
# channels; pairs), FP1 (not projected), FP0's projection of the known points and its chain (single tiles)
RPN_CASES = [
    _sa("rpn_sa3_ns16", 16, 1024, 256, 16, 256, [128, 196, 256], extra=256, off=0),
    _sa("rpn_sa3_ns32", 16, 1024, 256, 32, 256, [128, 196, 256], extra=256, off=256),
    _fp("rpn_fp1", 16, 4096, 1024, 512, 96, [256, 256]),
    _rows("rpn_fp0_projection", 16 * 4096, 256, [128], linear=True),
    _fp("rpn_fp0_chain", 16, 16384, 4096, 128, 1, [128, 128]),
]

CASES = [
    # tile counts: 5 tiles + 17 rows (odd count, the second tile of the last pair partial), one row, one partial tile,
    # 2 tiles + 1 row (the last pair's second tile empty)
    _rows("rows_337x33_160", 337, 33, [160], folded=False),
    _rows("rows_1x7_256_lin", 1, 7, [256], linear=True),
    _rows("rows_50x64_96_128", 50, 64, [96, 128], folded=False),
    _rows("rows_129x40_64_224_256", 129, 40, [64, 224, 256]),
    # K tails: a layer-0 chunk with 1, 2 or 3 K=8 steps of data
    _rows("rows_999x8_128_lin", 999, 8, [128], folded=False, linear=True),
    _rows("rows_640x81_256", 640, 81, [256]),
    _rows("rows2_500x5p8_b19p24_192", 500, 5, [192], a_pitch=8, a_off=0, c_b=19, b_pitch=24, b_off=4, folded=False),
    # SA: every centre size, 1-3 layers, widths on both pair builds; odd tile counts
    _sa("sa_ns4_f0_256", 2, 300, 35, 4, 0, [256], folded=False),
    _sa("sa_ns8_f1_32_64", 2, 400, 84, 8, 1, [32, 64], folded=False),
    _sa("sa_ns8_f9_160_lin", 2, 400, 84, 8, 9, [160], linear=True, extra=7, off=3),
    _sa("sa_ns16_f1_64_128", 3, 500, 63, 16, 1, [64, 128]),
    _sa("sa_ns16_f32_128_196_256", 2, 500, 33, 16, 32, [128, 196, 256], folded=False),
    _sa("sa_ns32_f3_64_96_128", 2, 500, 41, 32, 3, [64, 96, 128], folded=False),
    _sa("sa_ns32_f64_192_256", 2, 400, 21, 32, 64, [192, 256]),
    _sa("sa_ns64_f4_128", 3, 300, 21, 64, 4, [128]),
    _sa("sa_ns64_f20_96_224_lin", 2, 300, 13, 64, 20, [96, 224], folded=False, linear=True),
    _sa("sa_ns128_f5_64_128", 2, 400, 19, 128, 5, [64, 128]),
    _sa("sa_ns128_f40_128_256", 2, 300, 9, 128, 40, [128, 256], folded=False),
    # FP: with and without skip
    _fp("fp_k64_s0_128", 2, 333, 50, 64, 0, [128]),
    _fp("fp_k70_s5_96_128_lin", 2, 999, 300, 70, 5, [96, 128], folded=False, linear=True),
    _fp("fp_k256_s0_256_256", 2, 401, 100, 256, 0, [256, 256]),
    _fp("fp_k129_s33_160_96_lin", 3, 257, 64, 129, 33, [160, 96], folded=False, linear=True),
    # split chains: the last segment is a pair launch that reads the rows the <8,1> segment before it wrote
    _fp("fp_split_512_256_256", 2, 130, 40, 64, 16, [512, 256, 256], folded=False),
    _sa("sa_split_512_196_256", 2, 200, 17, 16, 13, [512, 196, 256]),
    _rows("rows_split_256_512_256_lin", 300, 100, [256, 512, 256], linear=True),
]


def _bits(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.int32), np.ascontiguousarray(b).view(np.int32))


def _run(case, cuda):
    chain, _, layers, inp = R.make(case)
    ref, bound = R.expected(case["kind"], chain, layers, inp)
    launch = Launch(case, chain, inp, cuda)
    outs = []
    for resident in (1, 0):
        label = "%s [mlp_resident=%d]" % (case["name"], resident)
        with C.options(mlp_resident=resident):
            flats = launch.run()
        launch.verify(flats, ref, bound, label)
        outs.append(flats)
    for x, y in zip(*outs):
        assert _bits(x, y), "%s: resident and streaming differ in %d words" % (case["name"], (x.view(np.int32) != y.view(np.int32)).sum())
    return launch


@pytest.mark.parametrize("case", RPN_CASES + CASES, ids=[c["name"] for c in RPN_CASES + CASES])
def test_stream_pair(cuda, case):
    _run(case, cuda)


@pytest.mark.parametrize("name", ["fp_k70_s5_96_128_lin", "fp_k256_s0_256_256", "fp_k129_s33_160_96_lin"])
def test_stream_pair_fp_without_point_major(cuda, name):
    """without out_pm the channel-major output keeps the same bits"""
    case = next(c for c in CASES if c["name"] == name)
    launch = _run(case, cuda)
    I, (flat, out) = launch.inp, launch.bufs[0]
    with C.options(mlp_resident=0):
        with_pm = launch.run()[0]
        flat.fill_(SENTINEL)
        C.check(launch.lib.prb_fp_interp_mlp_ws(case["b"], case["n"], case["m"], case["c_known"], case["c_skip"],
                                                C.ptr(I["known_pm"]), C.ptr(I["idx"]), C.ptr(I["weight"]),
                                                C.ptr(I["skip"]) if case["c_skip"] else None, ctypes.byref(launch.desc),
                                                C.ptr(out), None, C.ptr(launch.ws), C.c_size_t(launch.wsb), C.stream()),
                case["name"])
        torch.cuda.synchronize()
    assert _bits(flat.cpu().numpy(), with_pm)
