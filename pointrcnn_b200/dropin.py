"""Register the H100 implementations under the reference's import names.

    import pointrcnn_b200.dropin as dropin; dropin.activate()

After this, with the reference tree on sys.path, `lib/net/*.py` and `tools/*.py` import unchanged:
    import pointnet2_cuda / iou3d_cuda / roipool3d_cuda                    -> pointrcnn_b200.ext.*
    pointnet2_lib.pointnet2.{pointnet2_utils,pointnet2_modules,pytorch_utils} -> pointrcnn_b200.pointnet2.*
    lib.utils.iou3d.iou3d_utils, lib.utils.roipool3d.roipool3d_utils       -> pointrcnn_b200.{iou3d,roipool3d}.*
    lib.rpn.proposal_layer (ProposalLayer)                                 -> pointrcnn_b200.rpn.proposal_layer
    lib.rpn.proposal_target_layer (ProposalTargetLayer)                    -> pointrcnn_b200.rpn.proposal_target_layer
Optionally (compat=True) also provides the tiny stand-ins the 2019-era reference needs on a modern stack:
`easydict`, `tensorboardX.SummaryWriter` (no-op), `fire`, and a default Loader for `yaml.load`
(SURVEY.md section 0) -- none of them is on the operator path.
"""
import importlib
import sys
import types


def _alias(name, module):
    sys.modules[name] = module
    parent, _, child = name.rpartition(".")
    if parent:
        if parent not in sys.modules:
            pkg = types.ModuleType(parent)
            pkg.__path__ = []
            _alias(parent, pkg)
        setattr(sys.modules[parent], child, module)


def activate(compat=False):
    from .ext import iou3d_cuda, pointnet2_cuda, roipool3d_cuda
    _alias("pointnet2_cuda", pointnet2_cuda)
    _alias("iou3d_cuda", iou3d_cuda)
    _alias("roipool3d_cuda", roipool3d_cuda)
    if compat:
        _install_compat()
    from .pointnet2 import pointnet2_modules, pointnet2_utils, pytorch_utils
    for mod, name in ((pointnet2_utils, "pointnet2_utils"), (pointnet2_modules, "pointnet2_modules"),
                      (pytorch_utils, "pytorch_utils")):
        _alias("pointnet2_lib.pointnet2." + name, mod)
    # lib.utils.* must stay the reference's own package when its tree is importable: only the two wrapper
    # modules are replaced
    for pkg in ("lib", "lib.utils", "lib.utils.iou3d", "lib.utils.roipool3d"):
        try:
            importlib.import_module(pkg)
        except ImportError:
            m = types.ModuleType(pkg)
            m.__path__ = []
            _alias(pkg, m)
    from .iou3d import iou3d_utils
    from .roipool3d import roipool3d_utils
    _alias("lib.utils.iou3d.iou3d_utils", iou3d_utils)
    _alias("lib.utils.roipool3d.roipool3d_utils", roipool3d_utils)
    # next to the hot path (SURVEY.md section 8(f) rank 1): the RPN proposal layer, same class and signature
    try:
        importlib.import_module("lib.rpn")
    except ImportError:
        m = types.ModuleType("lib.rpn")
        m.__path__ = []
        _alias("lib.rpn", m)
    from .rpn import proposal_layer, proposal_target_layer
    _alias("lib.rpn.proposal_layer", proposal_layer)
    # rank 2: the RCNN target layer (one IoU launch per batch, batched jitter loop); lib/net/rcnn_net.py imports it by name
    _alias("lib.rpn.proposal_target_layer", proposal_target_layer)


def _install_compat():
    if "easydict" not in sys.modules:
        try:
            importlib.import_module("easydict")
        except ImportError:
            m = types.ModuleType("easydict")

            class EasyDict(dict):
                def __init__(self, d=None, **kw):
                    super().__init__()
                    for k, v in dict(d or {}, **kw).items():
                        self[k] = v

                def __setitem__(self, k, v):
                    if isinstance(v, dict) and not isinstance(v, EasyDict):
                        v = EasyDict(v)
                    elif isinstance(v, (list, tuple)):
                        v = type(v)(EasyDict(x) if isinstance(x, dict) and not isinstance(x, EasyDict) else x for x in v)
                    super().__setitem__(k, v)

                __setattr__ = __setitem__

                def __getattr__(self, k):
                    try:
                        return self[k]
                    except KeyError:
                        raise AttributeError(k)

            m.EasyDict = EasyDict
            sys.modules["easydict"] = m
    try:
        importlib.import_module("tensorboardX")
    except ImportError:
        m = types.ModuleType("tensorboardX")

        class SummaryWriter:
            def __init__(self, *a, **k):
                pass

            def __getattr__(self, name):
                return lambda *a, **k: None

        m.SummaryWriter = SummaryWriter
        sys.modules["tensorboardX"] = m
    try:
        importlib.import_module("fire")
    except ImportError:
        m = types.ModuleType("fire")
        m.Fire = lambda *a, **k: None
        sys.modules["fire"] = m
    import yaml
    if not getattr(yaml.load, "_prb_default_loader", False):
        _orig = yaml.load

        def load(stream, Loader=None, **kw):
            return _orig(stream, Loader=Loader or yaml.FullLoader, **kw)

        load._prb_default_loader = True
        yaml.load = load
