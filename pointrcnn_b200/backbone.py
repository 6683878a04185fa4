"""The RPN PointNet++ backbone wiring (mirror of lib/net/pointnet2_msg.py:6-70) parameterised by a plain
dict instead of the reference's global EasyDict, so benches and GPU tests can build it without the
reference tree.  Module / parameter names are the reference's (`SA_modules.k.mlps.i.layer{j}...`,
`FP_modules.k.mlp.layer{j}...`), so a reference checkpoint's backbone keys load as they are.
"""
import copy

import torch
import torch.nn as nn

from .pointnet2.pointnet2_modules import PointnetFPModule, PointnetSAModuleMSG

# tools/cfgs/default.yaml:38-51
RPN_DEFAULT = dict(
    USE_BN=True,
    NPOINTS=[4096, 1024, 256, 64],
    RADIUS=[[0.1, 0.5], [0.5, 1.0], [1.0, 2.0], [2.0, 4.0]],
    NSAMPLE=[[16, 32], [16, 32], [16, 32], [16, 32]],
    MLPS=[[[16, 16, 32], [32, 32, 64]], [[64, 64, 128], [64, 96, 128]], [[128, 196, 256], [128, 196, 256]],
          [[256, 256, 512], [256, 384, 512]]],
    FP_MLPS=[[128, 128], [256, 256], [512, 512], [512, 512]],
)


class Pointnet2MSG(nn.Module):
    def __init__(self, input_channels=0, use_xyz=True, cfg=None):
        super().__init__()
        cfg = copy.deepcopy(cfg or RPN_DEFAULT)
        self.SA_modules = nn.ModuleList()
        channel_in = input_channels
        skip_channel_list = [input_channels]
        channel_out = channel_in
        for k in range(len(cfg["NPOINTS"])):
            mlps = [list(m) for m in cfg["MLPS"][k]]
            channel_out = 0
            for i in range(len(mlps)):
                mlps[i] = [channel_in] + mlps[i]
                channel_out += mlps[i][-1]
            self.SA_modules.append(PointnetSAModuleMSG(npoint=cfg["NPOINTS"][k], radii=cfg["RADIUS"][k],
                                                       nsamples=cfg["NSAMPLE"][k], mlps=mlps, use_xyz=use_xyz, bn=cfg["USE_BN"]))
            skip_channel_list.append(channel_out)
            channel_in = channel_out
        self.FP_modules = nn.ModuleList()
        fp = cfg["FP_MLPS"]
        for k in range(len(fp)):
            pre_channel = fp[k + 1][-1] if k + 1 < len(fp) else channel_out
            self.FP_modules.append(PointnetFPModule(mlp=[pre_channel + skip_channel_list[k]] + list(fp[k])))
        self.FP_modules[0].emit_point_major = False   # the finest level feeds the heads, nothing gathers from it

    @staticmethod
    def _break_up_pc(pc):
        xyz = pc[..., 0:3].contiguous()
        features = pc[..., 3:].transpose(1, 2).contiguous() if pc.size(-1) > 3 else None
        return xyz, features

    def forward(self, pointcloud: torch.Tensor):
        xyz, features = self._break_up_pc(pointcloud)
        if self._plannable(xyz, features):
            return self._forward_planned(xyz, features)
        l_xyz, l_features = [xyz], [features]
        for sa in self.SA_modules:
            li_xyz, li_features = sa(l_xyz[-1], l_features[-1])
            l_xyz.append(li_xyz)
            l_features.append(li_features)
        for i in range(-1, -(len(self.FP_modules) + 1), -1):
            l_features[i - 1] = self.FP_modules[i](l_xyz[i - 1], l_xyz[i], l_features[i - 1], l_features[i])
        return l_xyz[0], l_features[0]

    # ------------------------------------------------------------------ stream-planned forward (eval / no_grad)
    # Everything geometric -- the four FPS levels, the ball queries, the 3-NN searches -- depends on the input
    # coordinates only.  The planned forward runs that chain on side streams and lets the feature MLPs (main stream)
    # follow it level by level: the FPS of level k+1 and all neighbour searches overlap the MLP of level k.
    # Same kernels, same results as the level-by-level loop.
    def _plannable(self, xyz, features):
        from . import config
        # opt-in: at batch 16 every kernel except the small FPS levels already fills the GPU, and the persistent MLP
        # CTAs queue behind the neighbour-search CTAs they share SMs with, so the side-stream plan is not the default.
        if not config.get("enable_plan") or not xyz.is_cuda:
            return False
        if not all(m._can_fuse(xyz, features, None) for m in self.SA_modules):
            return False
        probe = torch.empty(0, device=xyz.device)
        return all(m._can_fuse(xyz, xyz, None, probe) for m in self.FP_modules)

    def _forward_planned(self, xyz, features):
        dev = xyz.device
        main = torch.cuda.current_stream(dev)
        if getattr(self, "_streams", None) is None or self._streams[0].device != dev:
            self._streams = (torch.cuda.Stream(dev), torch.cuda.Stream(dev))
        s_fps, s_nbr = self._streams
        start = torch.cuda.Event()
        start.record(main)
        nlev = len(self.SA_modules)
        l_xyz = [xyz]
        ev_fps, ev_bq, geo = [], [], []
        # FPS chain on its own stream
        with torch.cuda.stream(s_fps):
            s_fps.wait_event(start)
            from .pointnet2 import pointnet2_utils as pu
            for sa in self.SA_modules:
                _, nx = pu.furthest_point_sample_xyz(l_xyz[-1], sa.npoint)
                nx.record_stream(main); nx.record_stream(s_nbr)
                e = torch.cuda.Event(); e.record(s_fps)
                l_xyz.append(nx); ev_fps.append(e)
        # neighbour searches on a second stream, each as soon as its centres exist
        with torch.cuda.stream(s_nbr):
            s_nbr.wait_event(start)
            for k, sa in enumerate(self.SA_modules):
                s_nbr.wait_event(ev_fps[k])
                _, centres, idxs, nss = sa.fused_geometry(l_xyz[k], l_xyz[k + 1])
                for t in idxs:
                    t.record_stream(main)
                e = torch.cuda.Event(); e.record(s_nbr)
                geo.append((centres, idxs, nss)); ev_bq.append(e)
            nn, ev_nn = {}, {}
            for i in range(-1, -(len(self.FP_modules) + 1), -1):
                lvl = nlev + i          # unknown level index (i=-1 -> nlev-1)
                idx, w = self.FP_modules[i].fused_geometry(l_xyz[lvl], l_xyz[lvl + 1])
                idx.record_stream(main); w.record_stream(main)
                e = torch.cuda.Event(); e.record(s_nbr)
                nn[i], ev_nn[i] = (idx, w), e
        # feature MLPs on the caller's stream
        l_features = [features]
        for k, sa in enumerate(self.SA_modules):
            main.wait_event(ev_bq[k])
            centres, idxs, nss = geo[k]
            l_features.append(sa.fused_mlp(l_xyz[k], l_features[k], centres, idxs, nss))
        for i in range(-1, -(len(self.FP_modules) + 1), -1):
            main.wait_event(ev_nn[i])
            idx, w = nn[i]
            l_features[i - 1] = self.FP_modules[i].fused_mlp(l_xyz[i - 1].size(1), idx, w, l_features[i - 1], l_features[i])
        return l_xyz[0], l_features[0]


def get_model(input_channels=0, use_xyz=True, cfg=None):
    return Pointnet2MSG(input_channels=input_channels, use_xyz=use_xyz, cfg=cfg)
