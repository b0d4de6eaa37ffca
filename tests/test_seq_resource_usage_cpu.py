"""The hashed-table (Bloom) sequence kernels compile without register spills (sm_90a).

Reads `cuobjdump --dump-resource-usage` of the built library (no GPU needed): every
instantiation the sequence step launches on a hashed item table -- seq_gather_hashed_kernel,
seq_score_kernel / mix_score_kernel / seq_reduce_kernel with HASHED = true at all six lane-group
widths, and pool_rep_kernel / pool_bwd_kernel reading by position at all three chunk counts --
must have no stack frame and no local memory."""
import pytest

from test_mf_resource_usage_cpu import _find, _usage

LPRS = (1, 2, 4, 8, 16, 32)
CASES = ([('seq_gather_hashed_kernel<%d>' % l, 'seq_gather_hashed_kernelILi%dEE' % l) for l in LPRS] +
         [('%s<%d,true>' % (k, l), '%sILi%dELb1EE' % (k, l))
          for k in ('seq_score_kernel', 'mix_score_kernel', 'seq_reduce_kernel') for l in LPRS] +
         [('%s<%d,true>' % (k, n), '%sILi%dELb1EE' % (k, n))
          for k in ('pool_rep_kernel', 'pool_bwd_kernel') for n in (1, 2, 4)])


@pytest.mark.parametrize('name,mangled', CASES, ids=[c[0] for c in CASES])
def test_hashed_sequence_kernels_do_not_spill(name, mangled):
    r = _find(_usage(), mangled)
    assert r['STACK'] == 0 and r['LOCAL'] == 0, '%s spills: %s' % (name, r)
