"""Sharded evaluation of sequence models on the CPU (gloo, worlds 1, 2 and 3, NumPy backend):
sequence_mrr_score, sequence_precision_recall_score and predict of a ShardedImplicitSequenceModel for
PoolNet, CNNNet, LSTMNet and MixtureLSTMNet against oracle/evaluation.py on the full tables.

The backend and the oracle build every representation one sequence at a time through the float64
oracles (oracle/seq.py, lstm.py, mixture.py) and every score with the same per-element float64
arithmetic (an ordered dot product, or oracle/mixture_eval.py), so a score does not depend on the
block, the rank's slice or the item shard it is computed in.  The results must then be equal, not
close.  Equal item rows on different shards give exact ties across shards."""

import numpy as np
import pytest
import torch

from oracle import evaluation as oev
from oracle import lstm as olstm
from oracle import mixture as omix
from oracle import mixture_eval as omev
from oracle import seq as oseq
from sharded_common import run_world
from test_sharded_eval_cpu import EvalNumpyBackend
from test_sharded_seq_cpu import LSTM_KEYS, SeqBackend

I, D, S, M = 13, 8, 7, 2            # world 3: items [0,5) [5,10) [10,13); world 2: [0,7) [7,13)
N, BLOCK = 9, 4                     # blocks of 4, 4 and 1 sequences
NETS = ['pooling', 'cnn', 'lstm', 'mixture']
PRED_IDS = np.array([12, 0, 1, 7, 7, 3, 9])
FLOAT_MAX = np.finfo(np.float32).max


def _f64(x):
    return (x.detach().numpy() if torch.is_tensor(x) else np.asarray(x)).astype(np.float64)


def _representations(E, seqs, cnn, lstm, mixture):
    """(n, S+1, width) float32 representations, each sequence through the float64 oracle on its own."""
    E = _f64(E)
    out = []
    for s in np.asarray(seqs):
        s = s.reshape(1, -1)
        if mixture is not None:
            proj = dict(w=_f64(mixture['w']), b=_f64(mixture['b']))
            r, _ = omix.mixture_representation(E, {k: _f64(lstm[k]) for k in LSTM_KEYS}, proj, s,
                                               int(mixture['num_mixtures']), np.float64)
        elif lstm is not None:
            r, _ = olstm.lstm_representation(E, {k: _f64(lstm[k]) for k in LSTM_KEYS}, s, np.float64)
        elif cnn is not None:
            convs = [(_f64(w), _f64(b)) for w, b in zip(cnn['weights'], cnn['biases'])]
            r, _ = oseq.cnn_representation(E, convs, s, cnn['kernel_width'], cnn['dilation'], cnn['nonlinearity'],
                                           cnn['residual'], np.float64)
        else:
            r, _ = oseq.pool_representation(E, s, np.float64)
        out.append(r[0])
    return np.stack(out).astype(np.float32)


def _dot(final, items, bias):
    """Dot-head scores, each element summed over d in order in float64, then + bias."""
    f, e = final.astype(np.float64), items.astype(np.float64)
    s = np.zeros((len(f), len(e)))
    for d in range(f.shape[1]):
        s += f[:, d:d + 1] * e[:, d]
    return (s + bias.astype(np.float64).reshape(1, -1)).astype(np.float32)


class SeqEvalBackend(SeqBackend):
    """NumPy stand-ins for GpuBackend's sequence-evaluation pieces."""

    rank_counts = EvalNumpyBackend.rank_counts

    def seq_representation(self, E_cache, seqs_idx, cnn, lstm, mixture):
        return torch.from_numpy(_representations(E_cache, seqs_idx.numpy(), cnn, lstm, mixture))

    def seq_dot_scores(self, final, items, item_bias):
        return torch.from_numpy(_dot(final.numpy(), items.numpy(), item_bias.numpy()))

    def mixture_scores(self, final, items, item_bias):
        s = omev.score_items(final.numpy(), items.numpy(), item_bias.numpy(), final.shape[1] // 2)
        return torch.from_numpy(s.astype(np.float32))

    def shard_mask_targets(self, scores, col_offset, excluded, row_ptr, targets):
        sc = scores.numpy()                         # the block itself: the overwrite is in place
        n_cols = sc.shape[1]
        if excluded is not None:
            for r, ids in enumerate(excluded.numpy()):
                c = ids - col_offset
                sc[r, c[(c >= 0) & (c < n_cols)]] = -FLOAT_MAX
        out = np.zeros(len(targets), np.float32)
        for r in range(len(row_ptr) - 1):
            for p in range(row_ptr[r], row_ptr[r + 1]):
                c = targets[p] - col_offset
                if 0 <= c < n_cols:
                    out[p] = sc[r, c]
        return torch.from_numpy(out)


def _net(kind):
    from spotlight_b200.sequence.representations import CNNNet, LSTMNet, MixtureLSTMNet, PoolNet
    torch.manual_seed(3)
    net = {'pooling': lambda: PoolNet(I, D),
           'cnn': lambda: CNNNet(I, D, kernel_width=[3, 2], dilation=[1, 2], num_layers=2),
           'lstm': lambda: LSTMNet(I, D),
           'mixture': lambda: MixtureLSTMNet(I, D, num_mixtures=M)}[kind]()
    with torch.no_grad():
        w, b = net.item_embeddings.weight, net.item_biases.weight
        b.copy_(torch.randn(I, 1) * 0.5)
        b[0] = 0
        for src, dst in ((1, 12), (3, 7)):          # equal rows on different shards
            w[dst], b[dst] = w[src], b[src]
    return net


def _sequences():
    rs = np.random.RandomState(8)
    seqs = rs.randint(1, I, (N, S)).astype(np.int64)
    for r in range(N):
        seqs[r, :rs.randint(0, S - 3)] = 0          # left padding
    seqs[0, -1] = seqs[0, 3]                        # targets that are prefix items
    seqs[1, -2] = seqs[1, 4]
    seqs[2, -1] = seqs[2, -2]                       # a repeated target among the last k
    seqs[4:8, -3:] = rs.randint(1, 5, (4, 3))       # block 1: every target on rank 0 (worlds 2 and 3)
    seqs[3, -1], seqs[5, -1], seqs[8, -1] = 12, 1, 7    # targets tied with an item on another shard
    return seqs


def _model(rank, world, dev, kind):
    from spotlight_b200.sharded import ShardedImplicitSequenceModel
    return ShardedImplicitSequenceModel(I, rank, world, dev, representation=_net(kind), embedding_dim=D,
                                        random_state=np.random.RandomState(0), backend=SeqEvalBackend())


def _eval_job(rank, world, dev, kind):
    from spotlight_b200.evaluation import sequence_mrr_score, sequence_precision_recall_score
    from spotlight_b200.interactions import SequenceInteractions
    model = _model(rank, world, dev, kind)
    seqs = _sequences()
    test = SequenceInteractions(seqs, num_items=I)
    # bad arguments raise on every rank before any collective, and leave the ranks in step
    bad = SequenceInteractions(np.concatenate([seqs[:2], [[0, 1, 2, 3, 4, 5, I]]]), num_items=I + 1)
    raised = []
    for call in (lambda: sequence_mrr_score(model, bad), lambda: sequence_precision_recall_score(model, bad, k=2),
                 lambda: sequence_precision_recall_score(model, test, k=S), lambda: model.predict(seqs[0], [0, I]),
                 lambda: model.predict([1, I, 2]), lambda: model.predict(seqs[0], [-1])):
        try:
            call()
        except ValueError:
            raised.append(True)
    out = {'raised': raised}
    for ex in (False, True):
        out['mrr', ex] = sequence_mrr_score(model, test, exclude_preceding=ex, sequence_block=BLOCK)
        for k in (1, 3):
            out['pr', k, ex] = sequence_precision_recall_score(model, test, k=k, exclude_preceding=ex,
                                                               sequence_block=BLOCK)
    out['predict all'] = model.predict(seqs[3])
    out['predict ids'] = model.predict(seqs[5, :-1], item_ids=PRED_IDS)
    return out


def _oracle_rows(kind, inputs):
    """(n, I) float32 scores of every item for the input sequences, on the full tables."""
    net = _net(kind)
    E = net.item_embeddings.weight.detach().numpy()
    bias = net.item_biases.weight.detach().numpy().reshape(-1)
    final = _representations(E, inputs, net._cnn_spec(), net._lstm_spec(), net._mixture_spec())[:, -1]
    if kind == 'mixture':
        return omev.score_items(final.reshape(len(final), 2 * M, D), E, bias, M).astype(np.float32)
    return _dot(final, E, bias)


@pytest.mark.parametrize('kind', NETS)
@pytest.mark.parametrize('world', [1, 2, 3])
def test_sharded_sequence_scorers_equal_the_oracle(world, kind):
    res = run_world(_eval_job, world, (kind,), timeout=240)
    seqs = _sequences()
    for rank in range(world):
        out = res[rank]
        assert out['raised'] == [True] * 6, rank
        for ex in (False, True):
            inputs = seqs[:, :-1]
            rows = _oracle_rows(kind, inputs)
            want = [1.0 / oev.average_rank(oev.exclude(r, x) if ex else r, t)
                    for r, x, t in zip(rows, inputs, seqs[:, -1])]
            assert np.array_equal(out['mrr', ex], want), (rank, ex)
            for k in (1, 3):
                inputs = seqs[:, :-k]
                rows = _oracle_rows(kind, inputs)
                wp, wr = oev.precision_recall(rows, list(seqs[:, -k:]), k, list(inputs) if ex else None,
                                              recall_denominator=k)
                p, r = out['pr', k, ex]
                assert p.shape == (N,) and np.array_equal(p, wp[:, 0]) and np.array_equal(r, wr[:, 0]), (rank, k, ex)
        assert out['predict all'].dtype == np.float32
        assert np.array_equal(out['predict all'], _oracle_rows(kind, seqs[3:4])[0]), rank
        assert np.array_equal(out['predict ids'], _oracle_rows(kind, seqs[5:6, :-1])[0, PRED_IDS]), rank
    for rank in range(1, world):                    # every rank has the whole result
        for key in res[0]:
            assert np.array_equal(np.asarray(res[rank][key]), np.asarray(res[0][key])), key


def test_fixture_has_the_cases_it_claims():
    """Exact ties across shards at targets, targets that are prefix items, a last block of one
    sequence (ranks with empty slices), a block whose targets only rank 0 owns at worlds 2 and 3, and
    hits and misses at k = 3 for every net."""
    from spotlight_b200.sharded import ShardPlan
    seqs = _sequences()
    assert N % BLOCK == 1
    assert any(t in row[:-1] for row, t in zip(seqs, seqs[:, -1]))
    assert any(set(row[-3:]) & set(row[:-3]) for row in seqs)
    for world in (2, 3):
        chunk = ShardPlan(1, I, world).ichunk
        assert (seqs[BLOCK:2 * BLOCK, -3:] < chunk).all()
        assert (seqs[:BLOCK, -1] >= chunk).any()
    for kind in NETS:
        rows = _oracle_rows(kind, seqs[:, :-1])
        assert (rows[:, 1] == rows[:, 12]).all() and (rows[:, 3] == rows[:, 7]).all()
        assert np.isin(seqs[:, -1], [1, 3, 7, 12]).sum() >= 3
        p, _ = oev.precision_recall(_oracle_rows(kind, seqs[:, :-3]), list(seqs[:, -3:]), 3, recall_denominator=3)
        assert 0 < p.sum() and (p == 0).any(), kind
