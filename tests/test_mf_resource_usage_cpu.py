"""The planned MF step's user and item kernels compile without register spills (sm_90a).

Reads `cuobjdump --dump-resource-usage` of the built library (no GPU needed): every
instantiation the step launches at D = 64 and 128 -- mf_user_kernel<LPR/2, 2, LOSS, 32> for all
six losses, mf_item_kernel<LPR, 32> and <LPR, 8> -- must have no stack frame and no local
memory, so none of their per-row loads or loop state goes through local memory."""
import functools
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, 'spotlight_b200', 'libspotlight_b200.so')
LOSSES = (0, 1, 2, 4, 5, 6)     # pointwise, bpr, hinge, regression, poisson, logistic


def _cuobjdump():
    exe = shutil.which('cuobjdump')
    if exe is None and os.path.exists('/usr/local/cuda/bin/cuobjdump'):
        exe = '/usr/local/cuda/bin/cuobjdump'
    return exe


@functools.lru_cache(maxsize=1)
def _usage():
    exe = _cuobjdump()
    if exe is None or not os.path.exists(LIB):
        pytest.skip('needs cuobjdump and the built library')
    txt = subprocess.run([exe, '--dump-resource-usage', LIB], capture_output=True, text=True,
                         check=True).stdout
    out, cur = {}, None
    for line in txt.splitlines():
        m = re.match(r'\s*Function (\S+):', line)
        if m:
            cur = m.group(1)
            continue
        m = re.match(r'\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)', line)
        if m and cur:
            out[cur] = {'REG': int(m.group(1)), 'STACK': int(m.group(2)), 'LOCAL': int(m.group(4))}
            cur = None
    return out


def _find(usage, mangled_args):
    hits = [v for k, v in usage.items() if mangled_args in k]
    assert len(hits) == 1, '%s: %d matches in the library' % (mangled_args, len(hits))
    return hits[0]


CASES = ([('mf_user_kernel<%d,2,%d,32>' % (lpr, loss), 'mf_user_kernelILi%dELi2ELi%dELi32EE' % (lpr, loss))
          for lpr in (8, 16) for loss in LOSSES] +
         [('mf_item_kernel<%d,%d>' % (lpr, ti), 'mf_item_kernelILi%dELi%dEE' % (lpr, ti))
          for lpr in (16, 32) for ti in (32, 8)])


@pytest.mark.parametrize('name,mangled', CASES, ids=[c[0] for c in CASES])
def test_planned_step_kernels_do_not_spill(name, mangled):
    r = _find(_usage(), mangled)
    assert r['STACK'] == 0 and r['LOCAL'] == 0, '%s spills: %s' % (name, r)
