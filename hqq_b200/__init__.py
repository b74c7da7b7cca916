"""hqq_b200 -- the HQQ quantize-and-infer hot path, written for NVIDIA H100 (sm_90a).

Public surface mirrors ``hqq.core``:

    from hqq_b200.core.quantize import HQQLinear, HQQBackend, BaseQuantizeConfig, Quantizer
    from hqq_b200.core.bitpack import BitPack
    from hqq_b200.core.optimize import optimize_weights_proximal

All arithmetic runs in ``libhqq_b200.so`` (hand-written CUDA behind a C ABI, see ``include/hqq_b200.h``);
build it with ``python -m hqq_b200.build``.  There is no CPU path and no alternative backend.
"""
__version__ = "0.1.0"

from . import _lib  # noqa: F401  (import does not load the .so; first use does)


def install_as_hqq() -> None:
    """Register this package's modules under the reference's import names (``hqq.core.quantize`` ...), so code
    written against mobiusml/hqq runs on the H100 path unchanged.  See INTEGRATION.md."""
    import sys
    import types

    from .core import bitpack, optimize, quantize, utils
    from .models import base as models_base
    from .models import hf as models_hf
    from .models.hf import base as models_hf_base

    def package(name):
        mod = types.ModuleType(name)
        mod.__path__ = []
        sys.modules[name] = mod
        return mod

    root, core, models = package("hqq"), package("hqq.core"), package("hqq.models")
    root.core, root.models = core, models
    for name, mod in (("quantize", quantize), ("bitpack", bitpack), ("optimize", optimize), ("utils", utils)):
        setattr(core, name, mod)
        sys.modules["hqq.core." + name] = mod
    models.base, models.hf = models_base, models_hf
    sys.modules["hqq.models.base"] = models_base
    sys.modules["hqq.models.hf"] = models_hf
    sys.modules["hqq.models.hf.base"] = models_hf_base
