"""flaxdiff_b200 - an H100-native (sm_90a) diffusion training / sampling engine with the
flaxdiff.schedulers / predictors / samplers / trainer / models.simple_unet.Unet API surface.

Host code is Python (PyTorch tensors as the container); all image- and activation-sized
arithmetic runs in the hand-written CUDA kernels of libfdx.so (include/fdx.h).  There is no
CPU or eager fallback: ops raise if the library is missing or tensors are not on a GPU.
"""
__version__ = "0.1.0"

from . import _defaults  # noqa: E402,F401  (kernel-generation defaults -> environment, before libfdx loads)
