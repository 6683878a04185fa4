"""pointrcnn_b200 -- H100 (sm_90a) kernels for PointRCNN's point-cloud operator path.

Layout
  csrc/      hand-written CUDA + the C ABI (include/pointrcnn_b200.h) -> libpointrcnn_b200.so
  _cabi.py   ctypes loader (fails loudly when the library is missing -- there is no CPU fallback)
  ext/       drop-in extension modules under the reference's names: pointnet2_cuda, iou3d_cuda, roipool3d_cuda
  pointnet2/ host-side mirror of pointnet2_lib/pointnet2/{pointnet2_utils,pointnet2_modules,pytorch_utils}.py
  iou3d/, roipool3d/  mirrors of lib/utils/{iou3d,roipool3d}/*_utils.py
  backbone.py  the RPN PointNet++ backbone wiring (lib/net/pointnet2_msg.py) for benches/tests
  dropin.py    registers all of the above under the reference's import names
"""
__version__ = "0.1.0"
