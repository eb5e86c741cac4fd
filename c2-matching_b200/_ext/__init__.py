"""Drop-in replacement for the reference's compiled top-level module `_ext`
(mmsr/models/archs/DCNv2/src/vision.cpp:3-8; imported as `import _ext as _backend` at
mmsr/models/archs/DCNv2/dcn_v2.py:6).  Same names, positional signatures and error behaviour;
the arithmetic runs in libc2m_sm100.so through the C ABI (include/c2m_sm100.h)."""
from c2m_b200.ops import (dcn_v2_backward, dcn_v2_forward, dcn_v2_psroi_pooling_backward,  # noqa: F401
                          dcn_v2_psroi_pooling_forward)
