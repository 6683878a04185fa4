"""oracle/make_golden_proposal_edges.py -- golden vectors of the RPN proposal path on the edge families of
tests/proposal_reference.py (range, argmax, heading-wrap, size, non-finite, quota and NMS edges).

Runs the reference's own decode_bbox_target and ProposalLayer on the CPU with the stand-ins of make_golden_proposal.py,
on every family without tied scores (a CPU and a CUDA sort need not order ties alike), and stores in
tests/golden/proposal_edges.npz, per case:
  <case>.decode              the first 512 decoded boxes (the NaN-argmax and heading-wrap semantics of the reference)
  <case>.<mode>_boxes/scores the proposals of each mode
  <case>.<mode>_raises       True where the reference stops (an empty near range: `assert i == 2`)
Usage (here, not on the GPU box):
    python oracle/make_golden_proposal_edges.py
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.append(os.path.join(ROOT, "oracle"))

import proposal_reference as PR  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "proposal_edges.npz")
DECODE_ROWS = 512


def cases():
    """(name, family, variant, n, seed, modes): quota scenes at 16384 points in the two axis-aligned modes, the others
    at 2048 points in TEST with both NMS types and score based"""
    out = []
    for i, (f, v) in enumerate(PR.SCENES):
        if f in PR.TIED:
            continue
        quota = f == "quota_edges"
        modes = ("test_normal", "train_normal") if quota else ("test_normal", "test_rotate", "score_based")
        out.append(("%s.%s" % (f, v or "all"), f, v, PR.N if quota else 2048, 100 + i, modes))
    return out


def main():
    from make_golden_proposal import install_reference
    ProposalLayer, cfg, decode_bbox_target = install_reference()
    out = {}
    for name, f, v, n, seed, modes in cases():
        scores, reg, xyz = PR.scene(f, v, n, seed)
        if f != "quota_edges":
            dec = decode_bbox_target(torch.from_numpy(xyz[:DECODE_ROWS]), torch.from_numpy(reg[:DECODE_ROWS]),
                                     anchor_size=torch.from_numpy(cfg.CLS_MEAN_SIZE[0]), loc_scope=cfg.RPN.LOC_SCOPE,
                                     loc_bin_size=cfg.RPN.LOC_BIN_SIZE, num_head_bin=cfg.RPN.NUM_HEAD_BIN,
                                     get_xz_fine=cfg.RPN.LOC_XZ_FINE, get_y_by_bin=False, get_ry_fine=False)
            out[name + ".decode"] = dec.numpy()
        for mode in modes:
            m = PR.MODES[mode]
            cfg.RPN.NMS_TYPE = m["nms_type"]
            cfg.TEST.RPN_DISTANCE_BASED_PROPOSE = m["distance_based"]
            layer = ProposalLayer(mode="TRAIN" if mode.startswith("train") else "TEST")
            try:
                with torch.no_grad():
                    b, s = layer(torch.from_numpy(scores[None]), torch.from_numpy(reg[None]), torch.from_numpy(xyz[None]))
            except AssertionError:
                out["%s.%s_raises" % (name, mode)] = np.array(True)
                print(name, mode, "raises")
                continue
            out["%s.%s_raises" % (name, mode)] = np.array(False)
            out["%s.%s_boxes" % (name, mode)] = b.numpy()[0]
            out["%s.%s_scores" % (name, mode)] = s.numpy()[0]
            print(name, mode, "rows:", int((s[0] != 0).sum()))
    np.savez_compressed(GOLDEN, **out)
    print("wrote", os.path.relpath(GOLDEN, ROOT), "%d bytes" % os.path.getsize(GOLDEN))


if __name__ == "__main__":
    main()
