"""gvd-b200: H100-native caption-decode hot path of grounded-video-description.

Layout:
  csrc/     hand-written sm_90a CUDA kernels + the C-ABI (include/gvd_b200.h)
  capi.py   ctypes binding of the C-ABI (raw device pointers, sizes, stream)
  misc/     host-side mirror of the reference's nn.Module surface
            (misc/AttModel.py, misc/model.py, misc/CaptionModelBU.py)
  synth.py  deterministic synthetic opt / weights / clip tensors
"""
__version__ = "0.1.0"
