"""The hashed-table sequence oracle (oracle/seq_bloom.py) and the cases of
tests/test_seq_bloom_oracle_gpu.py, checked without a GPU:

* oracle.seq_bloom reproduces the live reference's PoolNet + BloomEmbedding step
  (tests/golden/pool_pointwise_bloom.npz);
* with one hash onto a table of one row per id it is the plain-table oracle;
* every case exercises what it claims (seq_cases.check_properties and the hashing edges);
* the GPU tolerances catch every mutation of the oracle on those cases."""

import numpy as np
import pytest

from conftest import assert_close, load_golden
from oracle import seq_bloom as sb
from oracle.murmur import bloom_rows

GPU_TOL = dict(pos=1e-5, neg=1e-5, loss=1e-5, dW=2e-5, dbias=2e-5)


def test_pool_golden():
    g = load_golden('pool_pointwise_bloom')
    case = dict(net='pool', W=g['sd.item_embeddings.embeddings.weight'], H=int(g['bloom_H']),
                bias=g['sd.item_biases.weight'], seqs=g['seqs'], negs=g['negs'], loss='pointwise', n_neg=1,
                cnn=None)
    ref = sb.step(case)
    assert_close(ref['pos'], g['pos'], 1e-6, what='pos')
    assert_close(ref['neg'], g['neg'], 1e-6, what='neg')
    assert_close(ref['loss'], g['loss'], 1e-6, what='loss')
    assert_close(ref['dW'], g['grad.item_embeddings.embeddings.weight'], 1e-6, what='dW')
    assert_close(ref['dbias'], g['grad.item_biases.weight'], 1e-6, what='dbias')
    assert_close(sb.representation(case)[:, -1], g['final'], 1e-6, what='final')


@pytest.mark.parametrize('name', sb.GOLDEN)
def test_step_golden(name):
    """Bloom CNNNet (two layers, dilation), LSTMNet and MixtureLSTMNet steps of the live reference,
    with 2, 4 and 1 hashes on tables where ids collide."""
    from oracle.murmur import bloom_rows as br
    g = load_golden(name)
    case = sb.golden_case(g)
    ref, want = sb.step(case), sb.golden_grads(g)
    I, H, M = case['bias'].shape[0], case['H'], case['W'].shape[0]
    rows = br(np.arange(I), H, M)
    ids = np.unique(case['seqs'][case['seqs'] != 0])
    assert (rows[ids] == 0).any()
    if H >= 2:
        assert any(len(np.unique(rows[i])) < H for i in ids)
    assert_close(ref['pos'], g['pos'], 1e-6, what='pos')
    assert_close(ref['neg'], g['neg'].reshape(ref['neg'].shape), 1e-6, what='neg')
    assert_close(ref['loss'], g['loss'], 1e-6, what='loss')
    assert_close(ref['dW'], want['dW'], 1e-6, what='dW')
    assert_close(ref['dbias'], want['dbias'], 1e-6, what='dbias')
    for i, (dW, db) in enumerate(want.get('dconvs', [])):
        assert_close(ref['dconvs'][i][0], dW, 1e-6, what='dconv_w%d' % i)
        assert_close(ref['dconvs'][i][1], db, 1e-6, what='dconv_b%d' % i)
    for k, v in want.get('dlstm', {}).items():
        assert_close(ref['dlstm'][k], v, 1e-6, what='dlstm ' + k)
    for k, v in want.get('dmix', {}).items():
        assert_close(ref['dmix'][k], v, 1e-6, what='dmix ' + k)


@pytest.mark.parametrize('net', ['pool', 'cnn', 'lstm', 'mixture'])
def test_one_hash_on_a_permuted_table_is_the_plain_oracle(net):
    """H = 1 names one row per id; where the rows of the batch's ids are distinct and non-zero, the
    hashed step is the plain step on E = W[rows], its gradient moved to those rows."""
    case = sb.make_case(net, D=16, S=9, B=8, I=60, rows=200000, H=1, loss='bpr', seed=11)
    rows = bloom_rows(np.arange(60), 1, 200000)[:, 0]
    assert len(np.unique(rows[1:])) == 59 and (rows[1:] != 0).all()
    plain = dict(case, E=case['W'][rows])
    ref, pref = sb.step(case), sb._helpers(net).oracle_step(plain)
    assert_close(ref['pos'], pref['pos'], 1e-12, what='pos')
    assert_close(ref['dW'][rows[1:]], pref['dE'][1:], 1e-12, what='dW')
    assert_close(ref['dbias'], pref['dbias'], 1e-12, what='dbias')


@pytest.mark.parametrize('kw', sb.CASES, ids=[sb.case_id(k) for k in sb.CASES])
def test_case_properties(kw):
    case = sb.make_case(**kw)
    assert sb.check_properties(case, sb.step(case)) == []


def _caught(case, ref, mutate):
    bad = sb.step(case, mutate=(mutate,))
    for k, tol in GPU_TOL.items():
        a, e = np.asarray(bad[k], dtype=np.float64), np.asarray(ref[k], dtype=np.float64)
        if a.shape != e.shape or np.abs(a - e).max() > tol * np.abs(e).max():
            return True
    return False


@pytest.mark.parametrize('mutate', [m for m in sb.MUTATIONS if m != 'bias_with_rows'])
def test_mutations_caught(mutate):
    """Each restated kernel mistake moves an output of at least one GPU case beyond its tolerance."""
    hits = []
    for kw in sb.CASES:
        if mutate == 'neg_raw_id' and kw['net'] == 'mixture':
            continue
        case = sb.make_case(**kw)
        hits.append(_caught(case, sb.step(case), mutate))
    assert any(hits), '%s is not caught by any case' % mutate


def test_bias_with_rows_changes_the_fused_update():
    """A bias decayed with its rows: on the hinge cases some id whose terms all have gp = 0 has a row
    updated through the input role, so the fused test (weight decay on) sees its bias move."""
    hits = 0
    for kw in sb.CASES:
        case = sb.make_case(**kw)
        ref = sb.step(case)
        _, good = sb.updated(case, ref)
        _, bad = sb.updated(case, ref, ('bias_with_rows',))
        hits += int((bad & ~good & (case['bias'][:, 0] != 0)).sum())
    assert hits > 0


def test_updated_rows_cover_the_gradient():
    """Every row and bias with a gradient is updated; row 0 and the padding bias never are."""
    for kw in sb.CASES:
        case = sb.make_case(**kw)
        ref = sb.step(case)
        rows, ids = sb.updated(case, ref)
        assert not rows[0] and not ids[0]
        assert rows[(ref['dW'] != 0).any(axis=1)].all()
        assert ids[ref['dbias'][:, 0] != 0].all()
