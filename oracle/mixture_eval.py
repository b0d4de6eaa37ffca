"""MixtureLSTMNet all-items scoring (oracle).

TEST INFRASTRUCTURE ONLY.  Restates, in NumPy float64, what ``slb_mixture_scores`` computes:
``MixtureLSTMNet.forward`` (spotlight/sequence/representations.py:557-596) over every item, as the
per-sequence ``predict`` calls of spotlight/evaluation.py:59-151 score it, by calling
``oracle.mixture.head`` over all items.  Pinned against the live reference's predict rows in
tests/test_eval_mixture_oracle_cpu.py.
"""

import numpy as np

from oracle.mixture import head


def score_items(final_reps, E, beta, M):
    """Float64 scores (n, I) of every item for each final representation: ``head`` over all items.

    final_reps: (n, 2M, D) or the reference's (n, 2M, D, 1), blocks 0..M-1 the components c_m,
    M..2M-1 the mixture vectors v_m; E: (I, D) item rows; beta: (I,) or (I, 1) item biases."""
    P = np.asarray(final_reps, dtype=np.float64)
    n, D = P.shape[0], P.shape[2]
    P = P.reshape(n, 2 * M, D)
    E = np.asarray(E, dtype=np.float64)
    beta = np.asarray(beta, dtype=np.float64).reshape(-1)
    I = E.shape[0]
    out = np.empty((n, I))
    for r in range(n):                        # one row at a time bounds the (I, M, D) products
        c = np.broadcast_to(P[r, None, None, :M], (1, I, M, D))
        v = np.broadcast_to(P[r, None, None, M:], (1, I, M, D))
        out[r] = head(c, v, E[None], beta[None])[0][0]
    return out
