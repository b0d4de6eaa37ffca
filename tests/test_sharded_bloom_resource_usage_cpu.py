"""The kernels of the hashed-table step's users-only mode and of the owners' dense table step compile
without register spills (sm_90a).

Reads `cuobjdump --dump-resource-usage` of the built library (no GPU needed): every instantiation of
mf_bloom_users_prepass_kernel, mf_bloom_adam_users_kernel and adam_dense_table_kernel must have no
stack frame and no local memory."""
import pytest

from test_mf_resource_usage_cpu import _find, _usage

LPRS = (1, 2, 4, 8, 16, 32)
KERNELS = [('%s<%d>' % (k, l), '%sILi%dEE' % (k, l)) for k in
           ('mf_bloom_users_prepass_kernel', 'mf_bloom_adam_users_kernel', 'adam_dense_table_kernel') for l in LPRS]


@pytest.mark.parametrize('name,mangled', KERNELS, ids=[k[0] for k in KERNELS])
def test_sharded_bloom_kernels_do_not_spill(name, mangled):
    r = _find(_usage(), mangled)
    assert r['STACK'] == 0 and r['LOCAL'] == 0, '%s spills: %s' % (name, r)
