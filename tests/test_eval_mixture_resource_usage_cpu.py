"""The all-items mixture scoring kernel compiles without register spills (sm_90a).

Reads `cuobjdump --dump-resource-usage` of the built library (no GPU needed): every instantiation
of mixture_scores_kernel (M = 1 .. 8) must have no stack frame and no local memory, so its
2M dot products per pair stay in registers."""
import pytest

from test_mf_resource_usage_cpu import _find, _usage

KERNELS = [('mixture_scores_kernel<%d>' % m, 'mixture_scores_kernelILi%dEE' % m) for m in range(1, 9)]


@pytest.mark.parametrize('name,mangled', KERNELS, ids=[k[0] for k in KERNELS])
def test_mixture_scores_kernel_does_not_spill(name, mangled):
    r = _find(_usage(), mangled)
    assert r['STACK'] == 0 and r['LOCAL'] == 0, '%s spills: %s' % (name, r)
