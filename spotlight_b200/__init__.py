"""spotlight_b200 -- H100-native implicit-feedback training path behind the
maciejkula/spotlight model API.

Module paths mirror the reference (``spotlight.factorization.implicit`` ->
``spotlight_b200.factorization.implicit`` and so on) so existing code switches
by changing the import root.  The fit() inner loop runs in hand-written sm_90a
CUDA kernels reached through a C-ABI shared library (include/spotlight_b200.h);
there is no CPU path.
"""

__version__ = 'v0.1.0'
