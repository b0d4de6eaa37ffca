"""The generic route's kernels against the float64 oracle (oracle/embed.py): ``ops.embedding``,
``ops.embedding_backward``, ``ops.bloom_rows`` (csrc/embed.cu: emb_fwd_kernel, the segmented
scatter emb_bwd_kernel, bloom_rows_kernel), ``ops.mf_scores`` / ``ops.mf_scores_backward``
(csrc/mf.cu) and ``ops.pairwise_loss`` / ``ops.rating_loss`` (csrc/loss.cu).

Cases come from oracle/embed_cases.py: every (LPR, VEC4) width instantiation, segments around
seg_sort_cap and a row of 4096+ members, 0 to 24 hashes, compressed tables of 1 / 2 / 7 rows,
padding none / 0 / 5, n = 0, 1 and 2^20 + 5 at D = 1; scores with odd n, zero gradients, one
user owning the batch and the broadcast mode; losses up to 10^6 + 3 elements.

The lookup and its backward are bit-identical to the ordered float32 restatement (the kernels'
own addition order) and within 1e-6 of float64 plus the float32 summation bound; hashed rows are
integer-equal; scores, their gradients and the losses are within 1e-5 of float64; the backward,
the scores backward and the losses are bit-identical from one call to the next.
"""

import time

import numpy as np
import pytest
import torch

from conftest import assert_close
from oracle import embed as oe
from oracle import embed_cases as ec
from oracle.murmur import SEEDS

pytestmark = pytest.mark.gpu

MATRIX = ec.matrix()
LOOKUPS = [e for e in MATRIX if e[0] in ('segments', 'hashed', 'tiny', 'distinct', 'sized')]
HASHED = [e for e in LOOKUPS if e[0] in ('hashed', 'tiny') or (e[0] == 'sized' and e[2] > 0)]
SCORES = [e for e in MATRIX if e[0] == 'scores']
PAIRWISE = [e for e in MATRIX if e[0] == 'pairwise']
RATINGS = [e for e in MATRIX if e[0] == 'rating']
_CASES = {}


def case_of(entry):
    if entry not in _CASES:
        _CASES[entry] = ec.case_for(entry)
    return _CASES[entry]


def t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def host(x):
    return x.detach().cpu().numpy()


def seeds(H):
    return list(SEEDS[:H])


def bits_equal(a, b):
    a, b = np.ascontiguousarray(a, dtype=np.float32), np.ascontiguousarray(b, dtype=np.float32)
    return a.shape == b.shape and np.array_equal(a.view(np.int32), b.view(np.int32))


def _ids(entry):
    return [ec.entry_id(e) for e in entry]


# ------------------------------------------------------------------ lookups

@pytest.mark.parametrize('entry', LOOKUPS, ids=_ids(LOOKUPS))
def test_lookup_forward(entry):
    from spotlight_b200 import ops
    case = case_of(entry)
    got = host(ops.embedding(t(case['W']), t(case['ids']), seeds(case['H']), case['pad']))
    want = ec.ordered(case)['out']
    assert bits_equal(got, want), 'forward differs from the ordered float32 sums'
    assert ec.within(got, ec.oracle(case)['out'], ec.sum_bounds(case)['out']) is None


@pytest.mark.parametrize('entry', LOOKUPS, ids=_ids(LOOKUPS))
def test_lookup_backward(entry):
    from spotlight_b200 import ops
    case = case_of(entry)
    dout, ids = t(case['dout']), t(case['ids'])
    args = (seeds(case['H']), case['M'], case['pad'])
    t0 = time.perf_counter()
    got = ops.embedding_backward(dout, ids, *args)
    torch.cuda.synchronize()
    took = time.perf_counter() - t0
    again = ops.embedding_backward(dout, ids, *args)
    got, again = host(got), host(again)
    assert bits_equal(got, again), 'two calls differ'
    want = ec.ordered(case)['dW']
    bad = np.flatnonzero((got.view(np.int32) != want.view(np.int32)).any(axis=1))
    assert len(bad) == 0, 'rows %s differ from the ordered float32 sums (%d members)' % (
        bad[:8], oe.term_counts(case['ids'], case['H'], case['M'], case['pad'])[bad[0]])
    assert ec.within(got, ec.oracle(case)['dW'], ec.sum_bounds(case)['dW']) is None
    if case['pad'] >= 0:
        assert (got[case['pad']] == 0).all(), 'the frozen row has a gradient'
    print('%s: backward %.1f ms (first call)' % (ec.entry_id(entry), took * 1e3))


@pytest.mark.parametrize('entry', HASHED, ids=_ids(HASHED))
def test_bloom_rows(entry):
    from spotlight_b200 import ops
    case = case_of(entry)
    got = host(ops.bloom_rows(t(case['ids']), seeds(case['H']), case['M'], case['pad']))
    assert np.array_equal(got, oe.term_rows(case['ids'], case['H'], case['M'], case['pad']))


def test_backward_workspace_shared_across_widths():
    """Two tables with the same row count but other widths and batch sizes share the backward's
    workspace ('emb%d' % rows): alternating them, each call is still exact, so the segment
    index's counters are back at zero after every call."""
    from spotlight_b200 import ops
    rs = np.random.RandomState(7)
    M = 777
    cases = []
    for D, n, H in ((5, 3000, 0), (64, 900, 3), (1, 6000, 0)):
        ids = rs.randint(0, M if H == 0 else 10 ** 5, n).astype(np.int64)
        ids[:200] = 11                                   # a long segment
        cases.append(dict(D=D, H=H, pad=-1, M=M, ids=ids, W=ec.values(rs, (M, D)), dout=ec.values(rs, (n, D))))
    for case in cases + cases[::-1] + cases:
        got = host(ops.embedding_backward(t(case['dout']), t(case['ids']), seeds(case['H']), M, -1))
        assert bits_equal(got, ec.ordered(case)['dW'])


def test_autograd_through_layers():
    """ScaledEmbedding(padding_idx=3) and BloomEmbedding(padding_idx=5) forward and backward are the
    ops the tests above pin: the layer's .grad is the ordered float32 dW."""
    from spotlight_b200.layers import BloomEmbedding, ScaledEmbedding
    rs = np.random.RandomState(8)
    for layer, H, pad, M in ((ScaledEmbedding(50, 10, padding_idx=3), 0, 3, 50),
                             (BloomEmbedding(400, 6, compression_ratio=0.1, num_hash_functions=3, padding_idx=5),
                              3, 5, 40)):
        layer = layer.cuda()
        W = layer.weight if H == 0 else layer.embeddings.weight
        D = W.shape[1]
        with torch.no_grad():
            W.copy_(t(ec.values(rs, tuple(W.shape))))
        ids = rs.randint(0, 50 if H == 0 else 400, 700).astype(np.int64)
        ids[:9] = pad
        dout = ec.values(rs, (700, D))
        out = layer(t(ids)).reshape(700, D)
        out.backward(t(dout))
        case = dict(D=D, H=H, pad=pad, M=M, ids=ids, W=host(W), dout=dout)
        o = ec.ordered(case)
        assert bits_equal(host(out), o['out'])
        assert bits_equal(host(W.grad), o['dW'])


# ------------------------------------------------------------------ scores

@pytest.mark.parametrize('entry', SCORES, ids=_ids(SCORES))
def test_mf_scores(entry):
    from spotlight_b200 import ops
    case = case_of(entry)
    ref = ec.oracle(case)
    P = [t(case[k]) for k in ('Wu', 'Wi', 'bu', 'bi')]
    u, i = t(case['users']), t(case['items'])
    assert_close(host(ops.mf_scores(*P, u, i)), ref['scores'], 1e-5, what='scores')
    g = t(case['g'])
    outs = [[host(x) for x in ops.mf_scores_backward(g, P[0], P[1], u, i)] for _ in range(2)]
    for a, b in zip(*outs):
        assert bits_equal(a, b), 'two calls differ'
    for got, k in zip(outs[0], ('dWu', 'dWi', 'dbu', 'dbi')):
        assert_close(got, ref[k], 1e-5, what=k)


# ------------------------------------------------------------------ losses

@pytest.mark.parametrize('entry', PAIRWISE, ids=_ids(PAIRWISE))
def test_pairwise_loss(entry):
    from spotlight_b200 import _lib, ops
    case = case_of(entry)
    ref = ec.oracle(case)
    m = None if case['mask'] is None else t(case['mask'])
    outs = [[host(x) for x in ops.pairwise_loss(t(case['pos']), t(case['neg']), m, _lib.LOSS_KIND[case['loss']])]
            for _ in range(2)]
    for a, b in zip(*outs):
        assert bits_equal(a, b), 'two calls differ'
    for got, k in zip(outs[0], ('loss', 'gp', 'gn')):
        assert_close(got, ref[k], 1e-5, what=k)


@pytest.mark.parametrize('entry', RATINGS, ids=_ids(RATINGS))
def test_rating_loss(entry):
    from spotlight_b200 import _lib, ops
    case = case_of(entry)
    ref = ec.oracle(case)
    outs = [[host(x) for x in ops.rating_loss(t(case['pred']), t(case['ratings']), _lib.LOSS_KIND[case['loss']])]
            for _ in range(2)]
    for a, b in zip(*outs):
        assert bits_equal(a, b), 'two calls differ'
    assert_close(outs[0][0], ref['loss'], 1e-5, what='loss')
    assert_close(outs[0][1], ref['g'], 1e-5, what='g')


# ------------------------------------------------------------------ kernel names

def _width_picks():
    """One lookup width per (LPR, VEC4) instantiation of emb_fwd_kernel / emb_bwd_kernel."""
    picks = {}
    for e in LOOKUPS:
        if e[0] in ('segments', 'hashed'):
            picks.setdefault((oe.pow2_lanes(e[1]), oe.vec4(e[1])), e[1])
    return picks


def _profiled_lookup_kernel_names():
    """Kernel names of one lookup and one backward at each width of ``_width_picks``, as
    torch.profiler records them."""
    from torch.profiler import ProfilerActivity, profile
    from spotlight_b200 import ops
    rs = np.random.RandomState(9)
    small = [(t(ec.values(rs, (64, D))), t(rs.randint(0, 64, 100).astype(np.int64)), t(ec.values(rs, (100, D))))
             for D in _width_picks().values()]
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for W, ids, dout in small:
            ops.embedding(W, ids, [], -1)
            ops.embedding_backward(dout, ids, [], 64, -1)
        torch.cuda.synchronize()
    return sorted({ev.name.replace(' ', '') for ev in prof.events()
                   if ev.device_type == torch.autograd.DeviceType.CUDA})


def test_profiler_sees_every_width_variant():
    """The lookup widths launch emb_fwd_kernel and emb_bwd_kernel at all twelve (LPR, VEC4).  The
    profiling runs in a child process, so its profiler session does not share this process's CUPTI
    state with the other suites' profiler tests."""
    import json
    import os
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    code = ('import json, sys; sys.path.insert(0, %r); sys.path.insert(0, %r); '
            'import test_embed_oracle_gpu as m; print(json.dumps(m._profiled_lookup_kernel_names()))'
            % (os.path.dirname(here), here))
    out = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True, cwd=os.path.dirname(here),
                         timeout=600)
    assert out.returncode == 0, out.stderr[-4000:]
    names = json.loads(out.stdout.strip().split('\n')[-1])
    picks = _width_picks()
    assert len(picks) == 12
    for lanes, v in picks:
        for k in ('emb_fwd_kernel', 'emb_bwd_kernel'):
            w = '%s<%d,%s>' % (k, lanes, 'true' if v else 'false')
            assert any(w in n for n in names), (w, [n for n in names if 'emb_' in n])
