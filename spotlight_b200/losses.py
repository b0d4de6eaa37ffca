"""Loss functions with the reference's signatures (spotlight/losses.py), computed by
one fused CUDA kernel each way.

The implicit-feedback losses take ``(positive_predictions, negative_predictions,
mask=None)`` and return a 0-dim tensor: the mean of the per-element loss, or
``sum(loss * mask) / mask.sum()`` when a mask is given.  The explicit-feedback
losses take ``(observed_ratings, predicted_ratings)``.
"""

from spotlight_b200 import ops
from spotlight_b200.torch_utils import assert_no_grad


def pointwise_loss(positive_predictions, negative_predictions, mask=None):
    """Logistic loss: ``(1 - sigmoid(pos)) + sigmoid(neg)`` (losses.py:40-50)."""
    return ops.loss_op('pointwise', positive_predictions, negative_predictions, mask)


def bpr_loss(positive_predictions, negative_predictions, mask=None):
    """BPR: ``1 - sigmoid(pos - neg)`` (losses.py:82-90)."""
    return ops.loss_op('bpr', positive_predictions, negative_predictions, mask)


def hinge_loss(positive_predictions, negative_predictions, mask=None):
    """Hinge: ``max(neg - pos + 1, 0)`` (losses.py:115-124)."""
    return ops.loss_op('hinge', positive_predictions, negative_predictions, mask)


def adaptive_hinge_loss(positive_predictions, negative_predictions, mask=None):
    """Hinge against the highest of several negatives, ``negative_predictions``
    stacked on dim 0 (losses.py:164-166)."""
    return ops.loss_op('adaptive_hinge', positive_predictions, negative_predictions, mask)


# Explicit-feedback losses: ``(observed_ratings, predicted_ratings)``, the plain mean.

def regression_loss(observed_ratings, predicted_ratings):
    """Squared error ``(r - p)^2`` (losses.py:169-190)."""
    assert_no_grad(observed_ratings)
    return ops.rating_loss_op('regression', observed_ratings, predicted_ratings)


def poisson_loss(observed_ratings, predicted_ratings):
    """``p - r log p`` on the already exponentiated prediction ``p`` (losses.py:193-214)."""
    assert_no_grad(observed_ratings)
    return ops.rating_loss_op('poisson', observed_ratings, predicted_ratings)


def logistic_loss(observed_ratings, predicted_ratings):
    """Binary cross-entropy with logits against ``clamp(r, 0, 1)``, so -1/+1 ratings are
    0/1 targets (losses.py:217-244)."""
    assert_no_grad(observed_ratings)
    return ops.rating_loss_op('logistic', observed_ratings, predicted_ratings)
