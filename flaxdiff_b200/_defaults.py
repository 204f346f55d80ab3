"""Which kernel generation runs by default.  Every round-2 kernel has its round-1 predecessor one environment
switch away (DESIGN.md $6); this module turns a False below into that switch at import time, BEFORE libfdx is
loaded, so that reverting a kernel that misbehaves on some box is a one-word change and never a code edit in
the hot path.  An explicit environment variable always wins."""
import os

ROUND2_DEFAULTS = {
    # name: (enabled, environment variable that selects the predecessor)
    "fused_attention": (True, "FDX_ATTN_UNFUSED"),     # fdx_attention_fwd/bwd vs separate QK^T / softmax / PV launches
    # one-launch cluster GroupNorm backward vs the two-pass one: fewer resident warps per SM against one saved
    # re-read of x and dy; off by default, kept tested (tests/test_optin_kernels_gpu.py)
    "gn_cluster_bwd": (False, "FDX_GN_2PASS"),
    # bucketed all-reduce launched from the backward pass inside the training graph vs ONE fdx_comm call after it:
    # the NCCL CTAs take SMs from the persistent one-CTA-per-SM tensor-core kernels, which then need a second
    # wave.  Overlap stays available (FDX_NO_DP_OVERLAP=0).
    "dp_overlap": (False, "FDX_NO_DP_OVERLAP"),
}


def apply() -> None:
    for _name, (enabled, env) in ROUND2_DEFAULTS.items():
        if not enabled and env not in os.environ:
            os.environ[env] = "1"


apply()
