"""The one-pass target-ranking kernel compiles without register spills in both its instantiations
(sm_90a).

Reads `cuobjdump --dump-resource-usage` of the built library (no GPU needed): rank_targets_kernel for
slb_rank_targets (RankFinal) and for slb_rank_counts (RankCounts) must have no stack frame and no
local memory."""
import pytest

from test_mf_resource_usage_cpu import _find, _usage

KERNELS = [('rank_targets_kernel<%s>' % p, 'rank_targets_kernelINS_%d%sEEEv' % (len(p), p))
           for p in ('RankFinal', 'RankCounts')]


@pytest.mark.parametrize('name,mangled', KERNELS, ids=[k[0] for k in KERNELS])
def test_rank_targets_kernel_does_not_spill(name, mangled):
    r = _find(_usage(), mangled)
    assert r['STACK'] == 0 and r['LOCAL'] == 0, '%s spills: %s' % (name, r)
