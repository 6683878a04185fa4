"""The wgmma MLP chain through the C ABI against the float64 reference of mlp_reference.py, element by element.

Every case runs on the resident-weight kernel (prb_options.mlp_resident = 1, where the chain qualifies) and on the
streaming kernel (mlp_resident = 0).  Both runs must put every output element within its error bound, and they must
agree bit for bit.  Outputs are prefilled with a sentinel: whatever the kernel must not write (other channel slices of
the SA output, columns of a row output past its padded width, a guard behind every buffer) keeps it, and the padding
channels of row outputs are exactly zero.  Inputs the kernel must not read are NaN: the rows of xyz / feats_pm /
known_pm that no idx references, and the columns of a prb_mlp_rows2 buffer outside [:c_a] / [:c_b].
"""
import ctypes

import numpy as np
import pytest
import torch

import mlp_reference as R

pytestmark = pytest.mark.gpu

from pointrcnn_b200 import _cabi as C  # noqa: E402
from pointrcnn_b200.mlp_chain import Chain  # noqa: E402

SENTINEL = 7777.0
GUARD = 64          # floats behind every output buffer


def _dev(x, dev):
    return torch.from_numpy(np.ascontiguousarray(x)).to(dev)


def _out(shape, dev):
    """sentinel-filled buffer with a guard behind it: (flat tensor, view of the output part)"""
    n = int(np.prod(shape))
    flat = torch.full((n + GUARD,), SENTINEL, device=dev)
    return flat, flat[:n].view(shape)


class Launch:
    """device operands, descriptor and sentinel-filled outputs of one case; run() launches the chain once"""

    def __init__(self, case, chain, inp, dev):
        lib = C.lib()
        self.case, self.lib = case, lib
        self.chain = Chain(chain.kind, chain.split, chain.weights, chain.shift, chain.scale, chain.linear, dev)
        self.desc, self.co = self.chain.desc, self.chain.co
        self.L, self.C = len(chain.c_out), chain.c_out[-1]
        self.inp = {k: (_dev(v, dev) if isinstance(v, np.ndarray) else v) for k, v in inp.items()}
        k = case["kind"]
        if k == "sa":
            b, npoint = case["b"], case["npoint"]
            self.stride = self.C + case["extra"]
            self.bufs = [_out((b, self.stride, npoint), dev), _out((b, npoint, self.stride), dev)]
            wsb = lib.prb_sa_workspace_bytes(b, npoint, case["ns"], case["c_feat"], self.L, self.co)
        elif k == "fp":
            self.bufs = [_out((case["b"], self.C, case["n"]), dev), _out((case["b"], case["n"], self.C), dev)]
            wsb = lib.prb_fp_workspace_bytes(case["b"], case["n"], case["c_known"], case["c_skip"], self.L, self.co)
        else:
            self.np_last = R.round_up(self.C, 32)
            self.pitch = self.np_last + 8
            self.bufs = [_out((case["rows"], self.pitch), dev)]
            wsb = lib.prb_rows2_workspace_bytes(C.c_long(case["rows"]), case["c_a"], case.get("c_b", 0), self.L, self.co)
        self.wsb = wsb
        self.ws = torch.empty(max(wsb, 1), dtype=torch.uint8, device=dev)

    def run(self):
        """one launch from sentinel-filled outputs; returns the host copies of the flat buffers"""
        c, lib, I, d = self.case, self.lib, self.inp, ctypes.byref(self.desc)
        for flat, _ in self.bufs:
            flat.fill_(SENTINEL)
        if c["kind"] == "sa":
            rc = lib.prb_sa_group_mlp_max_ws(c["b"], c["n"], c["npoint"], c["ns"], c["c_feat"], C.ptr(I["xyz"]), C.ptr(I["new_xyz"]),
                                             C.ptr(I["feats_pm"]) if c["c_feat"] else None, C.ptr(I["idx"]), d,
                                             C.ptr(self.bufs[0][1]), C.ptr(self.bufs[1][1]), self.stride, c["off"], C.ptr(self.ws),
                                             C.c_size_t(self.wsb), C.stream())
        elif c["kind"] == "fp":
            rc = lib.prb_fp_interp_mlp_ws(c["b"], c["n"], c["m"], c["c_known"], c["c_skip"], C.ptr(I["known_pm"]), C.ptr(I["idx"]),
                                          C.ptr(I["weight"]), C.ptr(I["skip"]) if c["c_skip"] else None, d, C.ptr(self.bufs[0][1]),
                                          C.ptr(self.bufs[1][1]), C.ptr(self.ws), C.c_size_t(self.wsb), C.stream())
        elif "a_pitch" not in c:     # one contiguous input tensor: the plain entry point
            rc = lib.prb_mlp_rows(C.c_long(c["rows"]), c["c_a"], C.ptr(I["a"]), d, C.ptr(self.bufs[0][1]), self.pitch,
                                  C.ptr(self.ws), C.c_size_t(self.wsb), C.stream())
        else:
            a = ctypes.c_void_p(I["a"].data_ptr() + 4 * I["a_off"])
            b = ctypes.c_void_p(I["b"].data_ptr() + 4 * I["b_off"]) if "b" in I else None
            rc = lib.prb_mlp_rows2(C.c_long(c["rows"]), c["c_a"], a, c["a_pitch"], c.get("c_b", 0), b, c.get("b_pitch", 0), d,
                                   C.ptr(self.bufs[0][1]), self.pitch, C.ptr(self.ws), C.c_size_t(self.wsb), C.stream())
        C.check(rc, c["name"])
        torch.cuda.synchronize()
        return [flat.cpu().numpy() for flat, _ in self.bufs]

    def verify(self, flats, ref, bound, label):
        """every output element within its bound, everything else untouched; returns max err / bound"""
        c = self.case
        for flat in flats:
            assert (flat[-GUARD:] == SENTINEL).all(), "%s: written past the end of an output" % label
        if c["kind"] == "sa":
            b, npoint, off, C_ = c["b"], c["npoint"], c["off"], self.C
            out = flats[0][:-GUARD].reshape(b, self.stride, npoint)
            pm = flats[1][:-GUARD].reshape(b, npoint, self.stride)
            got = out[:, off:off + C_]
            outside = np.concatenate([out[:, :off].ravel(), out[:, off + C_:].ravel(), pm[:, :, :off].ravel(), pm[:, :, off + C_:].ravel()])
            assert (outside == SENTINEL).all(), "%s: channels outside the slice [%d, %d) were written" % (label, off, off + C_)
            assert np.array_equal(pm[:, :, off:off + C_], got.transpose(0, 2, 1)), "%s: the point-major twin differs" % label
        elif c["kind"] == "fp":
            got = flats[0][:-GUARD].reshape(c["b"], self.C, c["n"])
            pm = flats[1][:-GUARD].reshape(c["b"], c["n"], self.C)
            assert np.array_equal(pm, got.transpose(0, 2, 1)), "%s: the point-major twin differs" % label
        else:
            out = flats[0][:-GUARD].reshape(c["rows"], self.pitch)
            assert (out[:, self.np_last:] == SENTINEL).all(), "%s: columns past the padded width were written" % label
            assert (out[:, self.C:self.np_last] == 0).all(), "%s: padding channels are not exactly zero" % label
            got, ref, bound = out[:, :self.C], ref[:, :self.C], bound[:, :self.C]
        assert np.isfinite(got).all(), "%s: %d non-finite outputs" % (label, (~np.isfinite(got)).sum())
        ok, ratio, bad = R.check(got, ref, bound)
        assert ok, "%s: %d of %d elements outside the bound, max err/bound = %.3g" % (label, bad, got.size, ratio)
        return ratio


def _verify_case(case, dev, option_sets=({},)):
    lib = C.lib()
    chain, _, layers, inp = R.make(case)
    ref, bound = R.expected(case["kind"], chain, layers, inp)
    launch = Launch(case, chain, inp, dev)
    first, ratios = None, []
    for opts in option_sets:
        for resident in (1, 0):
            label = "%s [mlp_resident=%d%s]" % (case["name"], resident, "".join(", %s=%d" % kv for kv in opts.items()))
            with C.options(mlp_resident=resident, **opts):
                flats = launch.run()
            ratios.append(launch.verify(flats, ref, bound, label))
            if first is None:
                first = flats
            else:
                for x, y in zip(first, flats):
                    assert np.array_equal(x, y), "%s: differs from the resident default run, max |d| = %g" % (label, np.abs(x - y).max())
    print("%-32s %-34s max err/bound resident %.3f streaming %.3f" % (case["name"], case["build"], max(ratios[0::2]), max(ratios[1::2])))


@pytest.mark.parametrize("case", R.CASES, ids=[c["name"] for c in R.CASES])
def test_chain_within_bound(cuda, case):
    _verify_case(case, cuda)


@pytest.mark.parametrize("case", R.PERSIST_CASES, ids=[c["name"] for c in R.PERSIST_CASES])
def test_chain_persistent_ctas_within_bound(cuda, case):
    """a grid much smaller than the item count: each CTA (each resident warpgroup) walks hundreds of tiles, and the
    streaming kernel's weight ring wraps its phase bits many times; every grid size gives the same bits"""
    _verify_case(case, cuda, [{}] + R.PERSIST_OPTIONS)
