"""sfm-toy-library_b200: H100-native hot path of royshil/SfM-Toy-Library.

The product is the C-ABI shared library built from csrc/ (include/sfmb200.h); this Python package is the thin
host-side mirror of the reference's stage interface (stages.py), the ctypes binding (capi.py), the multi-GPU
plumbing over torch.distributed (dist.py) and the synthetic workloads (synth.py).
Import name: `sfm_toy_library_b200` (see sfm_toy_library_b200.py at the repo root).
"""
__version__ = "0.1.0"
