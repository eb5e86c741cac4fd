"""`feature_match_index` with the reference's signature (mmsr/models/archs/ref_map_util.py:26-86),
backed by the fused sm_90a correlation + argmax kernels.  No CPU path: the reference's CPU
arithmetic lives only in the test oracle."""
from c2m_b200.ops import feature_match_index  # noqa: F401


def sample_patches(inputs, patch_size=3, stride=1):
    """[C,h,w] -> [C,p,p,N] view of all sliding patches, row-major (ref_map_util.py:4-23).
    The H100 kernels never materialise this tensor; provided for API compatibility."""
    c = inputs.shape[0]
    u = inputs.unfold(1, patch_size, stride).unfold(2, patch_size, stride)
    return u.reshape(c, -1, patch_size, patch_size).permute(0, 2, 3, 1)
