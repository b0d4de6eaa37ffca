"""Sequence-step test cases and a NumPy restatement of the fused row-wise optimizers.

TEST INFRASTRUCTURE ONLY (tests/test_seq_oracle_gpu.py, tests/test_seq_oracle_cpu.py).

``make_case`` draws one PoolNet / CNNNet minibatch from a fixed seed, scaled so that the
case exercises the kernels: scores stay in the sigmoids' working range, 20-80 % of the
hinge-type positions are active, tanh does not saturate.  Unless switched off, every case
also carries the padding edges: a fully padded sequence, padding in the middle of a
sequence, the padding id drawn as a negative, and exact zeros inside embedding rows.
``check_properties`` verifies those scales on the float64 oracle's result.
"""

import numpy as np

from oracle import seq as oseq

LOSS_CYCLE = ('pointwise', 'bpr', 'hinge', 'adaptive_hinge')

# Conv geometries run on both conv paths (D = 32: mma.sync, D = 128: wgmma).  Together they take
# every kernel width in {1, 2, 5, 16}, dilation in {1, 3, a receptive field beyond S}, 1 / 3 / 8
# layers, residual on and off, tanh and relu, and S in {1, 2, 7, 9, 200}; B * (S + 1) leaves
# partial 64- and 128-row tiles (74, 104, 150, 603, 63, 402 rows).
GEOMETRIES = [
    dict(kernel_width=(1,), dilation=(1,), nonlinearity='tanh', residual=True, S=1, B=37),
    dict(kernel_width=(2, 5, 1), dilation=(1, 3, 1), nonlinearity='relu', residual=False, S=7, B=13),
    dict(kernel_width=(16,), dilation=(3,), nonlinearity='relu', residual=True, S=9, B=15),
    dict(kernel_width=(1, 2, 5, 16, 2, 1, 5, 2), dilation=(1, 3, 1, 1, 7, 1, 2, 1), nonlinearity='tanh',
         residual=True, S=200, B=3),
    dict(kernel_width=(2, 16), dilation=(5, 1), nonlinearity='tanh', residual=False, S=2, B=21),
    dict(kernel_width=(5, 1, 2), dilation=(250, 1, 3), nonlinearity='relu', residual=True, S=200, B=2),
]


def lpr_of(D):
    """Lanes per row of the sequence kernels (common.cuh lpr_for_dim): D / 4 rounded up to a power of two, <= 32."""
    l, p = D // 4, 1
    if l >= 32:
        return 32
    while p < l:
        p <<= 1
    return p


def seg_sort_cap(D):
    """Longest segment the reduce sorts in shared memory (segindex.cuh seg_sort_cap)."""
    G = lpr_of(D)
    return 128 if G >= 8 else (64 if G >= 4 else 16 * G)


def segment_lengths(case, ref):
    """Terms per item row of the gradient reduction: the target / input role at every unmasked
    position, plus each credited negative with a non-zero score gradient."""
    I = case['E'].shape[0]
    seqs = case['seqs']
    gn = ref['gn'].reshape(-1, *seqs.shape)
    negs = case['negs'].reshape(gn.shape)
    lens = np.bincount(seqs[seqs != oseq.PADDING_IDX], minlength=I)
    lens += np.bincount(negs[(gn != 0) & (negs != oseq.PADDING_IDX)], minlength=I)
    return lens


# E[max of n standard normals], n = 1..5: lifts the targets' biases over the hardest negative
_EMAX = {1: 0.0, 2: 0.5642, 3: 0.8463, 4: 1.0294, 5: 1.1630}


def make_case(net='pool', D=32, S=9, B=8, I=400, loss='bpr', n_neg=1, kernel_width=(3,),
              dilation=(1,), nonlinearity='tanh', residual=True, seed=0, padding=True,
              e0_nonzero=False, zero_frac=0.05, zipf=None, neg_tie=False):
    """One minibatch: dict(E, bias, seqs, negs, loss, n_neg, cnn=None | dict(...)).

    Targets come from items [1, I/2) and carry a bias lifted by 1 + E[max of n_neg normals],
    so the hinge margin is met at about half of the positions; negatives come from
    [I/2, I), one in ten from the whole table (rows shared by both roles).  ``zipf``: draw
    targets with P(item k) ~ k^-zipf (one item then holds most of them).  ``neg_tie``
    (adaptive hinge, n_neg >= 2): rows 1 and 2 of the negative range are bit-identical and
    are drawn together, in both orders, at a quarter of the positions.
    """
    rs = np.random.RandomState(seed)
    half = I // 2
    escale = np.sqrt(2.0 / D)                          # |e|^2 ~ 2 at any D
    E = (rs.randn(I, D) * escale).astype(np.float32)
    if zero_frac:
        E[rs.rand(I, D) < zero_frac] = 0.0
    E[0] = (rs.randn(D) * escale).astype(np.float32) if e0_nonzero else 0.0
    bias = rs.randn(I, 1).astype(np.float32)
    bias[1:half] += 1.0 + _EMAX[n_neg]
    bias[0] = rs.randn() if e0_nonzero else 0.0
    if zipf is None:
        seqs = rs.randint(1, half, (B, S)).astype(np.int64)
    else:
        seqs = np.minimum(rs.zipf(zipf, (B, S)), half - 1).astype(np.int64)
    n = n_neg if loss == 'adaptive_hinge' else 1
    negs = rs.randint(half, I, (n * B, S)).astype(np.int64)
    mix = rs.rand(n * B, S) < 0.1
    negs[mix] = rs.randint(0, I, int(mix.sum()))
    if padding:
        if B >= 3:
            seqs[0] = 0                                   # a fully padded sequence
        for b in range(1, B, 2):                          # left padding, as in the reference
            seqs[b, :rs.randint(0, S)] = 0
        if B >= 3 and S >= 3:                             # padding in the middle
            seqs[2, S // 3:(2 * S) // 3 + 1] = 0
        negs[rs.rand(n * B, S) < 0.03] = 0                # the padding id drawn as a negative
    if neg_tie:
        assert loss == 'adaptive_hinge' and n >= 2
        j1, j2 = half + 1, half + 2
        E[j2], bias[j2] = E[j1], bias[j1]
        bias[j1] = bias[j2] = bias[1:half].mean()
        n3 = negs.reshape(n, B, S)
        pick = rs.rand(B, S) < 0.25
        first = rs.rand(B, S) < 0.5
        n3[0][pick] = np.where(first, j1, j2)[pick]
        n3[1][pick] = np.where(first, j2, j1)[pick]
    case = dict(E=E, bias=bias, seqs=seqs, negs=negs, loss=loss, n_neg=n, cnn=None, net=net)
    if net == 'cnn':
        L = len(kernel_width)
        case['cnn'] = dict(kernel_width=[int(k) for k in kernel_width],
                           dilation=[int(d) for d in dilation], nonlinearity=nonlinearity,
                           residual=bool(residual))
        case['convs'] = _conv_weights(case, rs, L)
    return case


def _conv_weights(case, rs, L):
    """Per layer, scale W so the pre-activation's RMS is ~0.7 (tanh) / ~1 (relu) on this batch."""
    c = case['cnn']
    D = case['E'].shape[1]
    target = 0.7 if c['nonlinearity'] == 'tanh' else 1.0
    convs = []
    for l in range(L):
        k = c['kernel_width'][l]
        if l == 0:
            x = case['E'][case['seqs']].astype(np.float64)
        else:
            x, _ = oseq.cnn_representation(case['E'], convs, case['seqs'], c['kernel_width'][:l],
                                           c['dilation'][:l], c['nonlinearity'], c['residual'],
                                           np.float64)
        rms = max(float(np.sqrt((x ** 2).mean())), 1e-3)
        W = (rs.randn(D, D, k, 1) * (target / (rms * np.sqrt(k * D)))).astype(np.float32)
        b = (rs.randn(D) * 0.1 * target).astype(np.float32)
        convs.append((W, b))
    return convs


def oracle_step(case, dtype=np.float64, mutate=(), convs=None, negs=None, dilation=None):
    """oracle.seq.pool_step / cnn_step on a case (``convs`` / ``negs`` / ``dilation`` override)."""
    negs = case['negs'] if negs is None else negs
    if case['cnn'] is None:
        return oseq.pool_step(case['E'], case['bias'], case['seqs'], negs, case['loss'],
                              case['n_neg'], dtype, mutate)
    c = case['cnn']
    return oseq.cnn_step(case['E'], case['bias'], case['convs'] if convs is None else convs,
                         case['seqs'], negs, c['kernel_width'],
                         c['dilation'] if dilation is None else dilation, case['loss'],
                         case['n_neg'], c['nonlinearity'], c['residual'], dtype, mutate)


def oracle_representation(case, dtype=np.float64):
    """All S+1 positions of the representation, (B, S+1, D)."""
    if case['cnn'] is None:
        return oseq.pool_representation(case['E'], case['seqs'], dtype)[0]
    c = case['cnn']
    return oseq.cnn_representation(case['E'], case['convs'], case['seqs'], c['kernel_width'],
                                   c['dilation'], c['nonlinearity'], c['residual'], dtype)[0]


def check_properties(case, ref):
    """The case exercises the kernel: returns a list of violated properties (empty when fine)."""
    bad = []
    mask = case['seqs'] != oseq.PADDING_IDX
    if case['loss'] in ('hinge', 'adaptive_hinge') and mask.any():
        frac = float((ref['gp'][mask] != 0).mean())
        if not 0.2 <= frac <= 0.8:
            bad.append('hinge active at %.2f of the positions' % frac)
    if case['cnn'] is not None and case['cnn']['nonlinearity'] == 'tanh':
        c = case['cnn']
        _, saved = oseq.cnn_representation(case['E'], case['convs'], case['seqs'], c['kernel_width'],
                                           c['dilation'], c['nonlinearity'], c['residual'], np.float64)
        for l, (_, a) in enumerate(saved):
            sat = float((np.abs(a) > 0.99).mean())
            if sat > 0.01:
                bad.append('tanh of layer %d saturated at %.3f of the entries' % (l, sat))
    if case['loss'] in ('pointwise', 'bpr') and mask.any():
        far = float((np.abs(ref['pos'][mask]) > 6.0).mean())
        if far > 0.1:
            bad.append('%.2f of the scores beyond the sigmoid working range' % far)
    return bad


def updated_rows(case, ref):
    """Rows the fused optimizer updates: any term with a non-zero score gradient (target role
    at an unmasked position, or the credited negative), or a non-zero embedding gradient (the
    input role).  The padding row never is."""
    I = case['E'].shape[0]
    rows = np.zeros(I, dtype=bool)
    mask = case['seqs'] != oseq.PADDING_IDX
    rows[case['seqs'][mask & (ref['gp'] != 0)]] = True
    gn = ref['gn'].reshape(-1, *case['seqs'].shape)
    negs = case['negs'].reshape(gn.shape)
    rows[negs[gn != 0]] = True
    rows |= (ref['dE'] != 0).any(axis=1)
    rows[oseq.PADDING_IDX] = False
    return rows


def sgd(w, g, upd, lr, wd):
    """torch.optim.SGD (no momentum) on the entries where ``upd`` (broadcastable) is true."""
    w = w.astype(np.float64)
    d = g + wd * w
    return np.where(upd, w - lr * d, w)


def adagrad(w, state, g, upd, lr, wd, eps):
    """torch.optim.Adagrad (lr_decay 0) on the entries where ``upd`` is true -> (w, state)."""
    w = w.astype(np.float64)
    state = state.astype(np.float64)
    d = g + wd * w
    s_new = state + d * d
    w_new = w - lr * d / (np.sqrt(s_new) + eps)
    return np.where(upd, w_new, w), np.where(upd, s_new, state)
