"""The reference's `mmsr.models.archs.dcn` package (deformable convolution v1 / modulated, grouped) on the
project's own kernels; see deform_conv.py."""
from .deform_conv import (DeformConv, DeformConvPack, ModulatedDeformConv, ModulatedDeformConvPack, deform_conv,
                          modulated_deform_conv)

__all__ = [
    'DeformConv', 'DeformConvPack', 'ModulatedDeformConv', 'ModulatedDeformConvPack', 'deform_conv',
    'modulated_deform_conv'
]
