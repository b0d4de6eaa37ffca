"""The lazy-exact Adam kernels of the hashed-table MF step compile without register spills (sm_90a).

Reads `cuobjdump --dump-resource-usage` of the built library (no GPU needed): every instantiation
of mf_bloom_adam_prepass_kernel and mf_bloom_adam_apply_kernel, and bias_adam_apply_kernel, must have
no stack frame and no local memory."""
import pytest

from test_mf_resource_usage_cpu import _find, _usage

LPRS = (1, 2, 4, 8, 16, 32)
KERNELS = ([('mf_bloom_adam_prepass_kernel<%d>' % l, 'mf_bloom_adam_prepass_kernelILi%dEE' % l) for l in LPRS] +
           [('mf_bloom_adam_apply_kernel<%d>' % l, 'mf_bloom_adam_apply_kernelILi%dEE' % l) for l in LPRS] +
           [('bias_adam_apply_kernel<int>', 'bias_adam_apply_kernelIiEE')])


@pytest.mark.parametrize('name,mangled', KERNELS, ids=[k[0] for k in KERNELS])
def test_bloom_adam_kernels_do_not_spill(name, mangled):
    r = _find(_usage(), mangled)
    assert r['STACK'] == 0 and r['LOCAL'] == 0, '%s spills: %s' % (name, r)
