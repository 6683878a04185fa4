"""oracle/ref_backbone.py -- the reference's own CUDA-extension pipeline for the RPN backbone (B-ref of BASELINE.md):
the UNMODIFIED reference kernels (oracle/_ref, rebuilt for sm_90a) called in exactly the order
pointnet2_modules.py calls them (ref:pointnet2_modules.py:19-55,127-156, pointnet2_utils.py:241-264), with the
MLP through stock torch.nn Conv2d/BatchNorm2d/ReLU/max_pool2d (cuDNN/cuBLAS, torch defaults incl. TF32 convs).

TEST / BASELINE INFRASTRUCTURE ONLY: used by bench.py's `ref_cuda` comparator leg, oracle/bench_ref_cuda.py and the
end-to-end chain tests.  `net` is any module with the reference's structure (SA_modules[k].groupers/mlps/npoint,
FP_modules[k].mlp) -- e.g. pointrcnn_b200.backbone.Pointnet2MSG, whose parameters are the reference's.
"""
import torch
import torch.nn.functional as F

from . import refgpu as R

try:                                    # event timer only (per-family breakdown); optional
    from pointrcnn_b200 import prof
except Exception:                       # pragma: no cover
    import contextlib

    class prof:                         # noqa: N801
        region = staticmethod(lambda *a, **k: contextlib.nullcontext())

def sa_forward(mod, xyz, features):
    xyz_flipped = xyz.transpose(1, 2).contiguous()
    with prof.region("fps"):
        idx = R.fps(xyz, mod.npoint)
    with prof.region("gather"):
        new_xyz = R.gather(xyz_flipped, idx).transpose(1, 2).contiguous()
    outs = []
    for g, mlp in zip(mod.groupers, mod.mlps):
        with prof.region("ball_query"):
            bi = R.ball_query(g.radius, g.nsample, xyz, new_xyz)
        with prof.region("group"):
            xyz_trans = xyz.transpose(1, 2).contiguous()
            gx = R.group(xyz_trans, bi)
            gx -= new_xyz.transpose(1, 2).unsqueeze(-1)
            nf = torch.cat([gx, R.group(features, bi)], dim=1) if features is not None else gx
        with prof.region("sa_mlp"):
            nf = mlp(nf)
            nf = F.max_pool2d(nf, kernel_size=[1, nf.size(3)]).squeeze(-1)
        outs.append(nf)
    return new_xyz, torch.cat(outs, dim=1)


def fp_forward(mod, unknown, known, uf, kf):
    with prof.region("three_nn"):
        d2, idx = R.three_nn(unknown, known)
        dist = torch.sqrt(d2)
        recip = 1.0 / (dist + 1e-8)
        weight = recip / torch.sum(recip, dim=2, keepdim=True)
    with prof.region("interpolate"):
        interp = R.three_interpolate(kf, idx, weight)
    with prof.region("fp_mlp"):
        x = torch.cat([interp, uf], dim=1) if uf is not None else interp
        return mod.mlp(x.unsqueeze(-1)).squeeze(-1)


def backbone(net, pc):
    xyz = pc[..., 0:3].contiguous()
    feats = pc[..., 3:].transpose(1, 2).contiguous() if pc.size(-1) > 3 else None
    l_xyz, l_f = [xyz], [feats]
    for sa in net.SA_modules:
        nx, nf = sa_forward(sa, l_xyz[-1], l_f[-1])
        l_xyz.append(nx)
        l_f.append(nf)
    for i in range(-1, -(len(net.FP_modules) + 1), -1):
        l_f[i - 1] = fp_forward(net.FP_modules[i], l_xyz[i - 1], l_xyz[i], l_f[i - 1], l_f[i])
    return l_xyz[0], l_f[0]
