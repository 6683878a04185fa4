"""The device stage losses (csrc/stage_loss.cu through train.losses, impl="device") against the torch mirror of
get_rpn_loss / get_rcnn_loss, which tests/golden/stage_losses.npz pins to the reference's own functions.

Oracles: the mirror run on the CPU with float64 predictions (float32 labels, see _run) for values and gradients on
generic inputs; on inputs placed on the
mirror's kinks (logits of exactly 0, saturated sigmoids, smooth-L1 residuals of exactly +-1, shifts on bin edges and clamp
limits, headings at multiples of pi/2), the same mirror in float32 on the CPU: there float64 takes other branches than any
float32 run of the reference does (a saturated BCE, a heading of float32(pi/2) that float64 sees past pi/2)."""
import os
import sys

import numpy as np
import pytest
import torch

from pointrcnn_b200.rpn.stage import CLS_MEAN_SIZE
from pointrcnn_b200.train import losses as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _input_generators():
    """rpn_inputs / rcnn_inputs of oracle/make_golden_stage_losses.py, the golden's inputs.  Importing that module puts the
    reference checkout on sys.path (its main() runs the reference); the path is restored, nothing of the reference is read."""
    saved = list(sys.path)
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    try:
        import make_golden_stage_losses as G
    finally:
        sys.path[:] = saved
    return G.rpn_inputs, G.rcnn_inputs


rpn_inputs, rcnn_inputs = _input_generators()

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "stage_losses.npz")
MEAN = torch.from_numpy(CLS_MEAN_SIZE[0])
RPN_CLS = ("SigmoidFocalLoss", "DiceLoss", "BinaryCrossEntropy")
RCNN_CLS = ("BinaryCrossEntropy", "SigmoidFocalLoss", "CrossEntropy")
CE_WEIGHT = torch.tensor([1.0, 2.5, 0.7])


def _bce_same_dtype(input, target, *a, **kw):
    return _BCE(input, target.to(input.dtype), *a, **kw)


_BCE = torch.nn.functional.binary_cross_entropy


def _run(fn, cls, reg, rest, dtype, device, **kw):
    """loss and gradients of fn(cls, reg, *rest) with the predictions cast to dtype on device.  The labels stay float32, so a
    float64 run takes the bins and residual targets the reference computes (its float32 arithmetic) and differs from it only
    in the arithmetic on the predictions.  (The RCNN BCE term casts its labels with .float(); for a float64 run its target
    follows the input's dtype.)"""
    c, r = cls.to(device, dtype).requires_grad_(True), reg.to(device, dtype).requires_grad_(True)
    torch.nn.functional.binary_cross_entropy = _bce_same_dtype
    try:
        total, terms = fn(c, r, *[t.to(device) for t in rest], **kw)
    finally:
        torch.nn.functional.binary_cross_entropy = _BCE
    total.backward()
    return total, terms, c.grad, r.grad


def _rpn(cls, reg, lab, rl, impl, dtype, device, **kw):
    return _run(lambda c, r, lb, x, m: L.rpn_loss(c, r, lb, x, m, impl=impl, **kw), cls, reg, (lab, rl, MEAN), dtype, device)


def _rcnn(cls, reg, lab, valid, roi, gt, impl, dtype, device, **kw):
    if kw.get("loss_cls") == "CrossEntropy":
        kw = dict(kw, ce_weight=CE_WEIGHT.to(device=device, dtype=dtype))
    return _run(lambda c, r, lb, v, ro, g, m: L.rcnn_loss(c, r, lb, v, ro, g, m, impl=impl, **kw), cls, reg, (lab, valid, roi, gt, MEAN),
                dtype, device)


def _compare(dev, ref, rtol=1e-5, floor=1e-6):
    """values of every term the reference returns within rtol; gradients per element within rtol, with an absolute floor of
    floor x the tensor's largest magnitude"""
    total, terms, gc, gr = dev
    rtotal, rterms, rgc, rgr = ref
    assert set(rterms) <= set(terms), set(rterms) - set(terms)
    for k, v in rterms.items():
        assert v.dim() == 0 and terms[k].dim() == 0 and terms[k].is_cuda
        np.testing.assert_allclose(float(terms[k].detach()), float(v.detach()), rtol=rtol, atol=1e-7, err_msg=k)
    np.testing.assert_allclose(float(total.detach()), float(rtotal.detach()), rtol=rtol, atol=1e-7)
    for got, want, name in ((gc, rgc, "d cls"), (gr, rgr, "d reg")):
        got = got.double().cpu()
        want = torch.zeros_like(got) if want is None else want.double().cpu()        # the mirror's graph may not reach reg
        assert got.shape == want.shape
        bound = rtol * want.abs() + floor * float(want.abs().max())
        bad = (got - want).abs() > bound
        assert not bad.any(), "%s: %d elements off, worst %g at %s" % (name, int(bad.sum()), float(((got - want).abs() - bound).max()),
                                                                       torch.nonzero(bad)[:4].tolist())


def _rcnn_labels(name, lab):
    return lab.clamp(min=0) if name == "BinaryCrossEntropy" else lab


def _ce_inputs(cls, lab, seed=7):
    g = torch.Generator().manual_seed(seed)
    logits = torch.randn(cls.shape[0], 3, generator=g)
    lab = torch.where(lab > 0, torch.randint(1, 3, lab.shape, generator=g), lab)
    return logits, lab


@pytest.mark.parametrize("xz_fine", (True, False))
@pytest.mark.parametrize("name", RPN_CLS)
def test_rpn_values_and_gradients(cuda, name, xz_fine):
    cls, reg, lab, rl = rpn_inputs()
    if not xz_fine:
        reg = reg[..., :76 - 24]
    dev = _rpn(cls, reg, lab, rl, "device", torch.float32, cuda, loss_cls=name, loc_xz_fine=xz_fine)
    ref = _rpn(cls, reg, lab, rl, "torch", torch.float64, "cpu", loss_cls=name, loc_xz_fine=xz_fine)
    _compare(dev, ref)
    assert set(dev[1]) == set(ref[1])
    if xz_fine:      # the golden's configuration: within its bound of the reference's own get_rpn_loss
        t = dev[1]
        got = [float(dev[0]), float(t["rpn_loss_cls"]), float(t["rpn_loss_reg"]), float(t["loss_loc"]), float(t["loss_angle"]),
               3 * float(t["loss_size"])]
        np.testing.assert_allclose(got, np.load(GOLDEN)["rpn_%s" % name], rtol=3e-6, atol=1e-6)


@pytest.mark.parametrize("y_by_bin", (False, True))
@pytest.mark.parametrize("on_roi", (False, True))
@pytest.mark.parametrize("name", RCNN_CLS)
def test_rcnn_values_and_gradients(cuda, name, on_roi, y_by_bin):
    cls, reg, lab, valid, roi, gt = rcnn_inputs(C=53 if y_by_bin else 46)
    lab = _rcnn_labels(name, lab)
    if name == "CrossEntropy":
        cls, lab = _ce_inputs(cls, lab)
    kw = dict(loss_cls=name, size_res_on_roi=on_roi, loc_y_by_bin=y_by_bin)
    dev = _rcnn(cls, reg, lab, valid, roi, gt, "device", torch.float32, cuda, **kw)
    ref = _rcnn(cls, reg, lab, valid, roi, gt, "torch", torch.float64, "cpu", **kw)
    _compare(dev, ref)
    assert set(dev[1]) == set(ref[1])
    if name != "CrossEntropy" and not y_by_bin:
        want = np.load(GOLDEN)["rcnn_%s_%d" % (name, int(on_roi))]
        t = dev[1]
        np.testing.assert_allclose([float(dev[0]), float(t["rcnn_loss_cls"]), float(t["rcnn_loss_reg"])], want[:3], rtol=3e-6, atol=1e-6)


def _kink_rows(n, seed, C, nloc):
    """(cls, reg, lab, reg_label) of n rows on the mirror's kinks; rows 80.. are foreground"""
    g = torch.Generator().manual_seed(seed)
    cls = torch.randn(n, 1, generator=g)
    reg = torch.randn(n, C, generator=g) * 0.5
    lab = torch.tensor([-1, 0, 1])[torch.arange(n) % 3]
    cls[:40, 0] = 0.0                                                       # logits exactly 0
    cls[40:80, 0] = torch.tensor([25.0, -25.0, 30.0, -30.0, 21.0, -21.0, 120.0, -120.0]).repeat(5)    # saturated sigmoid
    lab[80:] = 1
    cls[80:120, 0] = torch.tensor([0.0, 25.0, -25.0, 30.0]).repeat(10)
    rl = torch.randn(n, 7, generator=g) * torch.tensor([1.0, 0.3, 1.0, 0.15, 0.15, 0.4, 1.5]) + torch.tensor([0, 0, 0, 1.5, 1.6, 3.9, 0.0])
    k = torch.arange(n - 80)
    edges = torch.cat([torch.arange(-3.0, 3.01, 0.5), torch.tensor([-3.5, -4.0, 3.0, 3.5, 4.0])])      # bin edges, both clamp limits
    rl[80:, 0] = edges[k % len(edges)]
    rl[80:, 2] = edges[(k + 5) % len(edges)]
    rl[80:, 1] = torch.tensor([0.25, -0.75, -0.25, -0.5, 0.5, 0.0, 1.0])[k % 7]
    ry = torch.tensor([0.0, np.pi / 2, np.pi, 1.5 * np.pi, 2 * np.pi, -np.pi / 2, -np.pi, -2 * np.pi])
    rl[80:, 6] = ry[k % len(ry)]
    rl[80::2, 3:6] = MEAN                                                    # size target exactly 0
    # residual predictions one away from targets that are exact: -0.5 on a bin edge, 0 for the heading at 0 (12 bins)
    reg[80::3, 2 * nloc:4 * nloc] = 0.5
    reg[81::3, 2 * nloc:4 * nloc] = -1.5
    return cls, reg, lab, rl


@pytest.mark.parametrize("name", RPN_CLS)
def test_rpn_gradients_on_kinks(cuda, name):
    cls, reg, lab, rl = _kink_rows(600, 11, 76, 12)
    reg[80::2, 48] = rl[80::2, 1] + 1.0                                      # y offset residual +1
    reg[81::2, 48] = rl[81::2, 1] - 1.0
    reg[80::4, 61:73] = 1.0                                                  # heading residual +-1 where its target is 0
    reg[82::4, 61:73] = -1.0
    reg[80::2, 73:76] = torch.tensor([1.0, -1.0, 1.0])                      # size residual +-1
    dev = _rpn(cls.view(1, -1, 1), reg.view(1, -1, 76), lab.view(1, -1), rl.view(1, -1, 7), "device", torch.float32, cuda, loss_cls=name)
    ref = _rpn(cls.view(1, -1, 1), reg.view(1, -1, 76), lab.view(1, -1), rl.view(1, -1, 7), "torch", torch.float32, "cpu", loss_cls=name)
    _compare(dev, ref)
    if name == "BinaryCrossEntropy":     # rows where the fp32 sigmoid is exactly 1 or 0: torch's BCE backward gives 0, not p - t
        sat = ((cls[:, 0] > 20) | (cls[:, 0] < -110)) & (lab >= 0)
        assert (dev[2].cpu().view(-1)[sat] == 0).all() and (ref[2].view(-1)[sat] == 0).all()
    if name == "SigmoidFocalLoss":       # logit exactly 0: clamp_min passes the gradient, abs does not
        z = (cls[:, 0] == 0) & (lab >= 0)
        assert (dev[2].cpu().view(-1)[z] != 0).all()


@pytest.mark.parametrize("y_by_bin", (False, True))
@pytest.mark.parametrize("name", RCNN_CLS)
def test_rcnn_gradients_on_kinks(cuda, name, y_by_bin):
    C = 53 if y_by_bin else 46
    cls, reg, lab, rl = _kink_rows(400, 12, C, 6)
    valid = (lab > 0).long()
    lab = _rcnn_labels(name, lab)
    if name == "CrossEntropy":
        cls, lab = _ce_inputs(cls, lab)
        cls[:40] = 0.0
    off = 24
    if y_by_bin:
        reg[80::3, off + 4:off + 8] = 0.5                                    # y on the bin edge -0.25: residual target -0.5
        off += 8
    else:
        reg[80::2, off] = rl[80::2, 1] + 1.0
        off += 1
    reg[80::2, off + 18:off + 21] = torch.tensor([1.0, -1.0, 1.0])
    roi = rl.clone()
    kw = dict(loss_cls=name, loc_y_by_bin=y_by_bin, size_res_on_roi=True)
    dev = _rcnn(cls, reg, lab, valid, roi, rl, "device", torch.float32, cuda, **kw)
    ref = _rcnn(cls, reg, lab, valid, roi, rl, "torch", torch.float32, "cpu", **kw)
    _compare(dev, ref)


def test_no_foreground_row(cuda):
    cls, reg, lab, rl = rpn_inputs()
    lab = lab.clamp(max=0)
    for name in RPN_CLS:
        total, terms, gc, gr = _rpn(cls, reg, lab, rl, "device", torch.float32, cuda, loss_cls=name)
        assert total.requires_grad and terms["rpn_loss_reg"].item() == 0.0
        assert all(terms[k].item() == 0.0 for k in L._reg_keys(True, False))
        assert torch.count_nonzero(gr).item() == 0
        assert (torch.count_nonzero(gc).item() > 0) == (name != "DiceLoss")      # Dice without a positive label is the constant 1
        _compare((total, terms, gc, gr), _rpn(cls, reg, lab, rl, "torch", torch.float64, "cpu", loss_cls=name))
    rc, rr, rlab, valid, roi, gt = rcnn_inputs()
    total, terms, gc, gr = _rcnn(rc, rr, rlab, torch.zeros_like(valid), roi, gt, "device", torch.float32, cuda, loss_cls="SigmoidFocalLoss")
    assert total.requires_grad and terms["rcnn_loss_reg"].item() == 0.0 and torch.count_nonzero(gr).item() == 0


def test_no_valid_row_and_a_single_row(cuda):
    cls, reg, lab, rl = rpn_inputs(B=1, N=50)
    for name in RPN_CLS:
        ignored = torch.full_like(lab, -1)
        _compare(_rpn(cls, reg, ignored, rl, "device", torch.float32, cuda, loss_cls=name),
                 _rpn(cls, reg, ignored, rl, "torch", torch.float64, "cpu", loss_cls=name))
        one = torch.ones(1, 1, dtype=torch.long)
        _compare(_rpn(cls[:, :1], reg[:, :1], one, rl[:, :1], "device", torch.float32, cuda, loss_cls=name),
                 _rpn(cls[:, :1], reg[:, :1], one, rl[:, :1], "torch", torch.float64, "cpu", loss_cls=name))
    rc, rr, rlab, valid, roi, gt = rcnn_inputs(R=40)
    for name in RCNN_CLS:
        c, lb = _ce_inputs(rc, rlab) if name == "CrossEntropy" else (rc, rlab)
        ignored = torch.full_like(lb, -1)
        _compare(_rcnn(c, rr, ignored, valid, roi, gt, "device", torch.float32, cuda, loss_cls=name),
                 _rcnn(c, rr, ignored, valid, roi, gt, "torch", torch.float64, "cpu", loss_cls=name))
        one = torch.ones(1, dtype=torch.long)
        _compare(_rcnn(c[:1], rr[:1], one, one, roi[:1], gt[:1], "device", torch.float32, cuda, loss_cls=name),
                 _rcnn(c[:1], rr[:1], one, one, roi[:1], gt[:1], "torch", torch.float64, "cpu", loss_cls=name))


def test_rpn_full_size(cuda):
    cls, reg, lab, rl = rpn_inputs(seed=401, B=16, N=16384)
    _compare(_rpn(cls, reg, lab, rl, "device", torch.float32, cuda), _rpn(cls, reg, lab, rl, "torch", torch.float64, "cpu"))


def test_bit_identical_repeats_and_no_host_synchronisation(cuda):
    cls, reg, lab, rl = (t.to(cuda) for t in rpn_inputs(seed=402, B=4, N=8192))
    rc, rr, rlab, valid, roi, gt = (t.to(cuda) for t in rcnn_inputs())
    mean = MEAN.to(cuda)
    ce_cls, ce_lab = (t.to(cuda) for t in _ce_inputs(rc.cpu(), rlab.cpu()))
    w = CE_WEIGHT.to(cuda)
    calls = [(cls, reg, lambda c, r, n=n: L.rpn_loss(c, r, lab, rl, mean, loss_cls=n, impl="device")) for n in RPN_CLS]
    calls += [(rc, rr, lambda c, r, n=n: L.rcnn_loss(c, r, rlab.clamp(min=0), valid, roi, gt, mean, loss_cls=n, size_res_on_roi=True,
                                                      impl="device")) for n in ("BinaryCrossEntropy", "SigmoidFocalLoss")]
    calls += [(ce_cls, rr, lambda c, r: L.rcnn_loss(c, r, ce_lab, valid, roi, gt, mean, loss_cls="CrossEntropy", ce_weight=w,
                                                     impl="device"))]

    def once(c0, r0, fn):
        c, r = c0.clone().requires_grad_(True), r0.clone().requires_grad_(True)
        total, terms = fn(c, r)
        total.backward()
        return [total.detach()] + [terms[k].detach() for k in sorted(terms)] + [c.grad, r.grad]

    for c0, r0, fn in calls:
        a = once(c0, r0, fn)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            b = once(c0, r0, fn)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_terms_carry_their_own_gradient(cuda):
    """backward through a single term (not the total) gives that term's gradient, as autograd of the mirror does"""
    cls, reg, lab, rl = rpn_inputs()
    for key in ("loss_x_bin", "loss_ry_res", "loss_size", "rpn_loss_cls", "loss_loc"):
        grads = []
        for impl, dt, dev in (("device", torch.float32, cuda), ("torch", torch.float64, "cpu")):
            c, r = cls.to(dev, dt).requires_grad_(True), reg.to(dev, dt).requires_grad_(True)
            total, terms = L.rpn_loss(c, r, lab.to(dev), rl.to(dev), MEAN.to(dev), impl=impl)
            (terms[key] * 2.0 + total).backward()
            grads.append((c.grad.double().cpu(), r.grad.double().cpu()))
        for got, want in zip(*grads):
            assert ((got - want).abs() <= 1e-5 * want.abs() + 1e-6 * want.abs().max()).all(), key


def test_rpn_trainer_with_the_device_loss_learns(cuda):
    import synth
    from pointrcnn_b200.train.step import RPNTrainer, synthetic_labels
    tr = RPNTrainer(input_channels=1, device=cuda, world=1, lr=0.002, seed=3, loss_impl="device")
    pc = torch.from_numpy(synth.u_kitti(2, 16384, 123, channels=4)).to(cuda)
    cls, reg = synthetic_labels(pc, seed=1)
    losses = []
    for _ in range(6):
        loss, terms = tr.step(pc, cls, reg, grad_norm_clip=1.0)
        losses.append(float(loss))
    assert all(np.isfinite(losses)) and losses[-1] < losses[0], losses
    assert {"rpn_loss_cls", "rpn_loss_reg", "loss_x_bin", "loss_ry_res", "loss_size"} <= set(terms)


def _jit_batch(cuda):
    from oracle import rcnn_offline as RO
    from pointrcnn_b200.datasets.rcnn_offline import RCNNOfflineSampler
    scenes = [RO.synth_scene(s, k, n_feat=128) for s, k in ((51, "mixed"), (52, "hard"))]
    return RCNNOfflineSampler(device=cuda).prepare_jit_batch(scenes)


def test_rcnn_step_jit_with_device_targets_and_loss_does_not_synchronise(cuda):
    from pointrcnn_b200.train.step import RCNNTrainer
    batch = _jit_batch(cuda)
    losses = {}
    for impl in ("torch", "device"):
        tr = RCNNTrainer(device=cuda, seed=5, target_draw="device", loss_impl=impl)
        torch.manual_seed(0)
        losses[impl] = float(tr.step_jit(batch)[0])
        if impl == "device":
            torch.cuda.synchronize()
            torch.cuda.set_sync_debug_mode("error")
            try:
                loss, terms = tr.step_jit(batch)
            finally:
                torch.cuda.set_sync_debug_mode(0)
            assert torch.isfinite(loss).item() and {"rcnn_loss_cls", "rcnn_loss_reg", "loss_ry_bin"} <= set(terms)
    np.testing.assert_allclose(losses["device"], losses["torch"], rtol=1e-5)
