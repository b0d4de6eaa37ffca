"""The shard-local exclusion and target read of the sharded sequence scorers compiles without register
spills (sm_90a).

Reads `cuobjdump --dump-resource-usage` of the built library (no GPU needed): shard_mask_targets_kernel
(slb_shard_mask_targets) must have no stack frame and no local memory."""

from test_mf_resource_usage_cpu import _find, _usage


def test_shard_mask_targets_kernel_does_not_spill():
    r = _find(_usage(), 'shard_mask_targets_kernelEPflllPKllS2_S2_S0_')
    assert r['STACK'] == 0 and r['LOCAL'] == 0, 'shard_mask_targets_kernel spills: %s' % r
