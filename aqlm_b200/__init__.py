"""aqlm_b200 -- H100-native (sm_90a) implementation of AQLM's quantized-linear hot path.

Mirrors the reference `aqlm` package surface (inference_lib/src/aqlm/__init__.py:1-3): `QuantizedLinear`,
`inference_kernels.{get_forward_pass_kernel,get_backward_pass_kernel,optimize_for_training}`, `utils.*`.
`install_as_aqlm()` aliases this package as `aqlm` in `sys.modules` so code that does `from aqlm import
QuantizedLinear` (Hugging Face's integration, the reference benchmarks) picks it up unchanged.
"""
import sys as _sys

from . import inference_kernels, utils  # noqa: F401
from .inference import QuantizedLinear  # noqa: F401
from .inference_kernels import optimize_for_training  # noqa: F401
from .inference_kernels import cuda_kernel as _cuda_kernel  # noqa: F401  (registers the aqlm:: ops; no JIT build)

from .grouped import QuantizedLinearGroup, ShardedQuantizedLinearGroup  # noqa: E402,F401
from .hf import fuse_shared_input_linears  # noqa: E402,F401
from .lora import LoraQuantizedLinear, add_lora, load_lora_adapter, save_lora_adapter  # noqa: E402,F401

__version__ = "1.1.6+b200.1"  # tracks the reference's aqlm 1.1.6 (inference_lib/setup.cfg:2-3); same string in pyproject.toml


def install_as_aqlm() -> None:
    """Make `import aqlm` resolve to this package (drop-in for the reference pip package)."""
    from . import inference
    from .inference_kernels import cuda_kernel, kernel_selector

    me = _sys.modules[__name__]
    _sys.modules["aqlm"] = me
    _sys.modules["aqlm.inference"] = inference
    _sys.modules["aqlm.utils"] = utils
    _sys.modules["aqlm.inference_kernels"] = inference_kernels
    _sys.modules["aqlm.inference_kernels.kernel_selector"] = kernel_selector
    _sys.modules["aqlm.inference_kernels.cuda_kernel"] = cuda_kernel
    _ensure_dist_metadata()


def _ensure_dist_metadata() -> None:
    """Hugging Face asks `importlib.metadata.version("aqlm")` (quantizer_aqlm.py:65, `is_trainable`).  A pip-installed
    copy of this repo provides that (pyproject.toml: distribution `aqlm`); when the package is used in-tree, expose the
    bundled `aqlm-<version>.dist-info` (aqlm_b200/_dist) on sys.path instead."""
    import os
    from importlib import metadata

    try:
        metadata.version("aqlm")
        return
    except metadata.PackageNotFoundError:
        pass
    dist_dir = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_dist")
    if os.path.isdir(dist_dir) and dist_dir not in _sys.path:
        _sys.path.append(dist_dir)
        import importlib

        importlib.invalidate_caches()
