"""`import aqlm` of an installed aqlm-b200 distribution.

The implementation lives in `aqlm_b200`; importing this shim aliases it (and its submodules) as `aqlm` in `sys.modules`,
so `from aqlm import QuantizedLinear`, `aqlm.inference_kernels.cuda_kernel.CUDA_KERNEL`, `aqlm.utils.*` (the reference's
import surface, inference_lib/src/aqlm/__init__.py:1-3) resolve to the H100-native code.  After this module has run,
`sys.modules["aqlm"]` IS `aqlm_b200` -- which is what the import statement returns.
"""
import aqlm_b200 as _impl

_impl.install_as_aqlm()
