"""c2m_b200 — host side of the H100-native C2-Matching restoration-forward hot path.

Python/PyTorch is plumbing (device memory, streams, torch.distributed); the arithmetic lives in
libc2m_sm100.so (csrc/, C ABI in include/c2m_sm100.h)."""
from .ops import (corr_argmax, dcn_v2_forward, dcn_v2_fused_forward, feature_match_index,  # noqa: F401
                  launch_count, offset_pyramid)
