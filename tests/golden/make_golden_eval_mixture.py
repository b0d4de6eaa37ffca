"""Generate the mixture-head evaluation golden fixture (tests/golden/eval_mixture.npz) from the
LIVE reference (build container only).

Run:  SPOTLIGHT_REFERENCE=<reference checkout> PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_eval_mixture.py

Imports the unmodified reference from the checkout SPOTLIGHT_REFERENCE names (read-only), builds
three small MixtureLSTMNet models with fixed, seeded weights -- ``representation='mixture'``
(M = 4), ``MixtureLSTMNet(num_mixtures=2)`` and a 3-taste net over a ``BloomEmbedding`` item
layer -- and records their state dicts, the sequences, the reference's ``predict`` rows and its
sequence_mrr_score / sequence_precision_recall_score outputs.  The tests read only the committed
fixture.
"""

import os
import sys

import numpy as np

sys.dont_write_bytecode = True
sys.path.insert(0, os.environ['SPOTLIGHT_REFERENCE'])

import torch  # noqa: E402

from spotlight.evaluation import sequence_mrr_score, sequence_precision_recall_score  # noqa: E402
from spotlight.interactions import SequenceInteractions  # noqa: E402
from spotlight.layers import BloomEmbedding  # noqa: E402
from spotlight.sequence.implicit import ImplicitSequenceModel  # noqa: E402
from spotlight.sequence.representations import MixtureLSTMNet  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
torch.set_num_threads(1)

I, D, N, S = 40, 8, 16, 8
KS = (1, 3)
# name -> (num_mixtures, Bloom (compression ratio, hashes) or None)
MODELS = {'mixture': (4, None), 'm2': (2, None), 'bloom': (3, (0.5, 2))}


def _state(net):
    return {'sd.' + k: v.detach().cpu().numpy().copy() for k, v in net.state_dict().items()}


def _separated(row):
    """No two scores of the row within 1e-4 of the row's largest magnitude: fp32 summation-order
    differences between implementations then cannot reorder the row."""
    s = np.sort(row.astype(np.float64))
    return bool(np.all(np.diff(s) > 1e-4 * np.abs(s).max()))


def _model(name, seqs, seed):
    M, bloom = MODELS[name]
    torch.manual_seed(seed)
    if name == 'mixture':
        rep = 'mixture'
    elif bloom is None:
        rep = MixtureLSTMNet(I, D, num_mixtures=M)
    else:
        emb = BloomEmbedding(I, D, compression_ratio=bloom[0], num_hash_functions=bloom[1], padding_idx=0)
        rep = MixtureLSTMNet(I, D, num_mixtures=M, item_embedding_layer=emb)
    m = ImplicitSequenceModel(representation=rep, embedding_dim=D, random_state=np.random.RandomState(seed))
    m._initialize(SequenceInteractions(seqs, num_items=I))
    net = m._net
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        # item rows and a projection large enough that the mixture weights are far from uniform
        table = net.item_embeddings.embeddings if bloom is not None else net.item_embeddings
        table.weight.copy_(torch.randn(table.weight.shape, generator=g) * 0.5)
        table.weight[0] = 0.0
        net.projection.weight.mul_(4.0)
        b = torch.randn(net.item_biases.weight.shape, generator=g) * 0.1
        b[0] = 0.0
        net.item_biases.weight.copy_(b)
    return m


def eval_mixture_case():
    rs = np.random.RandomState(31)

    def draw(n):
        row = rs.randint(1, I, S).astype(np.int32)
        if n % 3 == 0:
            row[:rs.randint(1, S - 3)] = 0                          # leading padding
        if n == 1:
            row[2] = row[-1]                                        # a target inside its own input
        if n == 2:
            row[-2] = row[-1]                                       # a repeated target
        return row

    seqs = np.stack([draw(n) for n in range(N)])
    models = {name: _model(name, seqs, 40 + j) for j, name in enumerate(MODELS)}
    for n in range(N):                                             # redraw rows holding a near-tie
        for _ in range(100):
            if all(_separated(m.predict(seqs[n, :-k])) for m in models.values() for k in KS):
                break
            seqs[n] = draw(n)
        assert all(_separated(m.predict(seqs[n, :-k])) for m in models.values() for k in KS), n
    out = dict(num_items=np.int64(I), dim=np.int64(D), seqs=seqs)
    inter = SequenceInteractions(seqs, num_items=I)
    for name, m in models.items():
        M, bloom = MODELS[name]
        out['%s.num_mixtures' % name] = np.int64(M)
        if bloom is not None:
            out['%s.bloom' % name] = np.array(bloom, dtype=np.float64)
        out.update({'%s.%s' % (name, k): v for k, v in _state(m._net).items()})
        for k in KS:
            out['%s.scores.k%d' % (name, k)] = np.stack([m.predict(seqs[n, :-k]) for n in range(N)])
        for ex in (False, True):
            out['%s.mrr.ex%d' % (name, ex)] = sequence_mrr_score(m, inter, exclude_preceding=ex)
            for k in KS:
                p, r = sequence_precision_recall_score(m, inter, k=k, exclude_preceding=ex)
                out['%s.pr.ex%d.k%d.p' % (name, ex, k)], out['%s.pr.ex%d.k%d.r' % (name, ex, k)] = p, r
    np.savez_compressed(os.path.join(HERE, 'eval_mixture.npz'), **out)


if __name__ == '__main__':
    eval_mixture_case()
