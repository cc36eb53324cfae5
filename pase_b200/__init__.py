"""pase_b200 -- H100-native (sm_90a) implementation of the PASE/PASE+ hot path.

Drop-in for the reference's ``pase.models.frontend.wf_builder`` /
``pase.models.pase.pase`` API (see INTEGRATION.md); all compute runs in the
hand-written CUDA kernels of ``pase_b200/csrc`` behind the C-ABI declared in
``include/pase_b200.h``.
"""
from .frontend import wf_builder, WaveFe            # noqa: F401
from .modules import Model, Saver, select_output    # noqa: F401

__version__ = "0.1.0"
