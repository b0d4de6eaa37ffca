"""Sequence step on a hashed (Bloom) item table, in float64 (oracle).

TEST INFRASTRUCTURE ONLY (tests/test_seq_bloom_oracle_cpu.py, tests/test_seq_bloom_oracle_gpu.py).

A ``BloomEmbedding`` item layer (spotlight/layers.py:132-244) passed to PoolNet / CNNNet / LSTMNet /
MixtureLSTMNet as ``item_embedding_layer`` (representations.py:68-72):

* item id i is the vector  e~(i) = sum_{k<H} W[h_k(i)],  h_k = oracle.murmur.bloom_rows
  (murmur3_32 of int32(i) with SEEDS[k], floor-mod M = int(ratio * num_items)); the padding id 0
  maps to row 0 for every hash;
* row 0 of W receives no gradient (padding_idx=0 of the table);
* the biases stay ZeroEmbedding(num_items, 1), indexed by the raw id.

``step`` forms the virtual table E~ = [e~(i)] for every id, runs the plain-table oracles on it
(oracle.seq.pool_step / cnn_step, oracle.lstm.lstm_step, oracle.mixture.mixture_step, through their
case helpers) and folds dE~ back onto W once per hash, dropping row 0.  An id whose hashes name one
row twice credits that row twice (the reference's ``.sum(1)`` backward).  dbias is the plain one.

Fused row-wise optimizers (``updated``):

* a table row is updated when it is not row 0 and either one of its terms has a non-zero score
  gradient (a position whose input id hashes onto it with gp != 0, or a credited negative with
  gn != 0) or its summed gradient is non-zero -- the plain sequence rule;
* a bias is updated when one of its terms has a non-zero score gradient -- the MF Bloom rule
  (oracle/bloom.py); a bias whose terms all have zero score gradient is not decayed.

``mutate`` restates plausible kernel mistakes (names below); tests/test_seq_bloom_oracle_cpu.py
shows the GPU tolerances catch each one on the GPU cases:

* ``'pad_hashed'``       the padding id hashed like any other id;
* ``'frozen_trained'``   row 0 trained (terms of real ids hashing onto it kept);
* ``'dup_once'``         a row named by two hashes of one id credited once;
* ``'first_hash'``       only the first hash read and trained;
* ``'mean'``             the mean of the hashed rows instead of the sum;
* ``'neg_raw_id'``       the credited negative's table gradient keyed by its raw id (mod M);
* ``'bias_by_row'``      the bias gradient keyed by the id's first hashed row;
* ``'bias_with_rows'``   (fused) a bias updated whenever one of its id's rows is updated.
"""

import numpy as np

from oracle import lstm_cases as lc
from oracle import mixture_cases as mc
from oracle import seq_cases as sc
from oracle.murmur import SEEDS, bloom_rows

PADDING_IDX = 0
MUTATIONS = ('pad_hashed', 'frozen_trained', 'dup_once', 'first_hash', 'mean', 'neg_raw_id',
             'bias_by_row', 'bias_with_rows')


def rows_of(num_items, H, M, mutate=()):
    """(num_items, H) hashed rows of every id (row 0 for the padding id)."""
    rows = bloom_rows(np.arange(num_items), H, M, PADDING_IDX if 'pad_hashed' not in mutate else -1)
    return rows[:, :1] if 'first_hash' in mutate else rows


def virtual_table(W, num_items, H, mutate=()):
    """E~ (num_items, D), float64: the summed (or, mutated, averaged / first) hashed rows of every id."""
    rows = rows_of(num_items, H, W.shape[0], mutate)
    E = W.astype(np.float64)[rows].sum(axis=1)
    return E / H if 'mean' in mutate else E


def fold(dE, num_items, H, M, mutate=()):
    """d loss / d W from d loss / d E~: each id's gradient onto each of its hashed rows."""
    rows = rows_of(num_items, H, M, mutate)
    dW = np.zeros((M, dE.shape[1]), dtype=np.float64)
    if 'dup_once' in mutate:
        for i in range(num_items):
            for r in np.unique(rows[i]):
                dW[r] += dE[i]
    else:
        for k in range(rows.shape[1]):
            np.add.at(dW, rows[:, k], dE)
    if 'mean' in mutate:
        dW /= H
    if 'frozen_trained' not in mutate:
        dW[PADDING_IDX] = 0.0
    return dW


def _helpers(net):
    return {'pool': sc, 'cnn': sc, 'lstm': lc, 'mixture': mc}[net]


def _virtual_case(case, mutate=()):
    v = dict(case)
    v['E'] = virtual_table(case['W'], case['bias'].shape[0], case['H'], mutate)
    return v


def representation(case, dtype=np.float64):
    """The representation at all S+1 positions, as the plain oracles give it on E~."""
    return _helpers(case['net']).oracle_representation(_virtual_case(case), dtype)


def _neg_role(case, ref, vcase):
    """d loss / d E~ of the credited negatives alone (PoolNet / CNNNet / LSTMNet: gn * r_t)."""
    rep = _helpers(case['net']).oracle_representation(vcase, np.float64)
    S = case['seqs'].shape[1]
    r = rep[:, :S]
    gn = ref['gn'].reshape(-1, *case['seqs'].shape)
    negs = case['negs'].reshape(gn.shape)
    out = np.zeros(vcase['E'].shape, dtype=np.float64)
    for k in range(gn.shape[0]):
        np.add.at(out, negs[k].reshape(-1), (gn[k][..., None] * r).reshape(-1, r.shape[-1]))
    out[PADDING_IDX] = 0.0
    return out


def step(case, dtype=np.float64, mutate=()):
    """One minibatch on the hashed table: the plain oracle's result with dE~ replaced by dW (M, D)."""
    vcase = _virtual_case(case, mutate)
    ref = dict(_helpers(case['net']).oracle_step(vcase, dtype))
    I, H, M = case['bias'].shape[0], case['H'], case['W'].shape[0]
    dE = ref.pop('dE')
    if 'neg_raw_id' in mutate:
        assert case['net'] != 'mixture', 'neg_raw_id restates the gn * r negative rows'
        dn = _neg_role(case, ref, vcase)
        dW = fold(dE - dn, I, H, M, mutate)
        raw = np.arange(I) % M
        np.add.at(dW, raw, dn)
        dW[PADDING_IDX] = 0.0
    else:
        dW = fold(dE, I, H, M, mutate)
    ref['dW'] = dW
    if 'bias_by_row' in mutate:
        db = np.zeros_like(ref['dbias'])
        np.add.at(db[:, 0], rows_of(I, H, M)[:, 0] % I, ref['dbias'][:, 0])
        db[PADDING_IDX] = 0.0
        ref['dbias'] = db
    return ref


def updated(case, ref, mutate=()):
    """(table rows, bias ids) the fused optimizer updates, boolean masks (M,) and (num_items,)."""
    I, H, M = case['bias'].shape[0], case['H'], case['W'].shape[0]
    rows = bloom_rows(np.arange(I), H, M)
    seqs = case['seqs']
    gn = ref['gn'].reshape(-1, *seqs.shape)
    negs = case['negs'].reshape(gn.shape)
    ids = np.concatenate([seqs[(seqs != PADDING_IDX) & (ref['gp'] != 0)], negs[gn != 0]])
    ids = ids[ids != PADDING_IDX]
    trow = np.zeros(M, dtype=bool)
    trow[rows[ids].ravel()] = True
    trow |= (ref['dW'] != 0).any(axis=1)
    trow[PADDING_IDX] = False
    bid = np.zeros(I, dtype=bool)
    bid[ids] = True
    if 'bias_with_rows' in mutate:
        touched = np.unique(np.concatenate([seqs[seqs != PADDING_IDX], negs[gn != 0]]))
        bid[touched[trow[rows[touched]].any(axis=1)]] = True
    bid[PADDING_IDX] = False
    return trow, bid


def make_case(net='pool', D=32, S=9, B=8, I=400, rows=60, H=4, loss='bpr', n_neg=1, seed=0, w0_nonzero=True, **kw):
    """One minibatch of ``net`` ('pool', 'cnn', 'lstm', 'mixture') on a hashed (rows, D) table with H
    hashes: the plain case (seq_cases / lstm_cases / mixture_cases make_case, whose padding edges it
    keeps) with its item table replaced by W, drawn so that an item's summed row has the plain
    case's scale.  ``w0_nonzero``: row 0 holds values (the forward reads it, nothing trains it)."""
    if net in ('pool', 'cnn'):
        case = sc.make_case(net, D=D, S=S, B=B, I=I, loss=loss, n_neg=n_neg, seed=seed, **kw)
    else:
        case = _helpers(net).make_case(D=D, S=S, B=B, I=I, loss=loss, n_neg=n_neg, seed=seed, **kw)
    rs = np.random.RandomState(seed + 31337)
    W = (rs.randn(rows, D) * np.sqrt(2.0 / D / H)).astype(np.float32)
    W[rs.rand(rows, D) < 0.05] = 0.0
    # the padding id sums row 0 H times: H * W[0] at the scale of one item
    W[PADDING_IDX] = (rs.randn(D) * np.sqrt(2.0 / D) / H).astype(np.float32) if w0_nonzero else 0.0
    case['W'], case['H'] = W, H
    case['seeds'] = SEEDS[:H]
    case['E'] = virtual_table(W, I, H).astype(np.float32)     # for helpers that size from E
    if net == 'cnn':                                          # conv scales measured on E~
        case['convs'] = sc._conv_weights(case, np.random.RandomState(seed + 7), len(case['cnn']['kernel_width']))
    return case


# The op-level cases of tests/test_seq_bloom_oracle_gpu.py that tests/test_seq_bloom_oracle_cpu.py
# also runs the mutations on: every representation and loss, 1 to 24 hashes, small tables where ids
# collide (and land on row 0), the conv / LSTM lane-group widths.  ``kw`` of make_case.
CASES = [
    dict(net='pool', D=32, S=20, B=16, rows=40, H=4, loss='pointwise', seed=1),
    dict(net='pool', D=12, S=20, B=16, rows=30, H=2, loss='hinge', seed=2),
    dict(net='cnn', D=32, S=20, B=16, rows=40, H=4, loss='bpr', kernel_width=(3, 2), dilation=(1, 2), seed=3),
    dict(net='cnn', D=128, S=20, B=8, rows=50, H=2, loss='adaptive_hinge', n_neg=5, kernel_width=(3,),
         dilation=(1,), seed=4),
    dict(net='lstm', D=32, S=20, B=16, rows=40, H=4, loss='adaptive_hinge', n_neg=5, seed=5),
    dict(net='lstm', D=16, S=20, B=16, rows=150, H=24, loss='pointwise', seed=6),
    dict(net='mixture', D=32, S=20, B=16, rows=40, H=4, loss='hinge', M=4, seed=7),
    dict(net='mixture', D=16, S=20, B=16, rows=60, H=1, loss='bpr', M=2, seed=8),
]


GOLDEN = ('seq_bloom_cnn_bpr', 'seq_bloom_lstm_adaptive', 'seq_bloom_mixture_pointwise')


def golden_case(g):
    """The case of a live-reference step fixture (tests/golden/make_golden_seq_bloom.py)."""
    net, H = str(g['net']), int(g['bloom_H'])
    case = dict(net=net, W=g['sd.item_embeddings.embeddings.weight'], H=H, seeds=SEEDS[:H],
                bias=g['sd.item_biases.weight'], seqs=g['seqs'], negs=g['negs'], loss=str(g['loss_name']),
                n_neg=int(g['n_neg']) if str(g['loss_name']) == 'adaptive_hinge' else 1, cnn=None)
    if net == 'cnn':
        case['cnn'] = dict(kernel_width=[3, 2], dilation=[1, 2], nonlinearity='tanh', residual=True)
        case['convs'] = [(g['sd.cnn_%d.weight' % i], g['sd.cnn_%d.bias' % i]) for i in range(2)]
    else:
        case['lstm'] = {k: g['sd.lstm.%s_l0' % v] for k, v in
                        (('w_ih', 'weight_ih'), ('w_hh', 'weight_hh'), ('b_ih', 'bias_ih'), ('b_hh', 'bias_hh'))}
    if net == 'mixture':
        case['M'] = 4
        case['proj'] = dict(w=g['sd.projection.weight'], b=g['sd.projection.bias'])
    return case


def golden_grads(g):
    """The fixture's gradients under the oracle's names: dW, dbias, dconvs / dlstm / dmix."""
    out = dict(dW=g['grad.item_embeddings.embeddings.weight'], dbias=g['grad.item_biases.weight'])
    net = str(g['net'])
    if net == 'cnn':
        out['dconvs'] = [(g['grad.cnn_%d.weight' % i], g['grad.cnn_%d.bias' % i]) for i in range(2)]
    else:
        out['dlstm'] = {k: g['grad.lstm.%s_l0' % v] for k, v in
                        (('w_ih', 'weight_ih'), ('w_hh', 'weight_hh'), ('b_ih', 'bias_ih'), ('b_hh', 'bias_hh'))}
    if net == 'mixture':
        out['dmix'] = dict(w=g['grad.projection.weight'], b=g['grad.projection.bias'])
    return out


def case_id(kw):
    return '%s-d%d-h%d-%s' % (kw['net'], kw['D'], kw['H'], kw['loss'])


def check_properties(case, ref):
    """The plain case's scale checks on E~, plus the hashing edges the case claims: a real id in the
    batch on row 0, and (H >= 2) an id in the batch with two hashes on one row."""
    bad = _helpers(case['net']).check_properties(_virtual_case(case), ref)
    I, H, M = case['bias'].shape[0], case['H'], case['W'].shape[0]
    rows = bloom_rows(np.arange(I), H, M)
    ids = np.unique(np.concatenate([case['seqs'].ravel(), case['negs'].ravel()]))
    ids = ids[ids != PADDING_IDX]
    if not (rows[ids] == PADDING_IDX).any():
        bad.append('no id of the batch hashes onto the frozen row')
    if H >= 2 and not any(len(np.unique(rows[i])) < H for i in ids):
        bad.append('no id of the batch has two hashes on one row')
    return bad
