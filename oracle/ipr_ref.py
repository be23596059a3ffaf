"""ORACLE: improved precision and recall restated in numpy fp64 (reference scripts/improved_precision_recall.py:
196-256).  Every term is fp64, |y|^2 included (the reference sums the subject's |y|^2 in the features' own dtype;
see DESIGN.md).  Dense N x N matrices: small inputs only."""
import numpy as np


def pairwise_distances(X, Y=None):
    """(distances, number of negative squared distances set to 0) as compute_pairwise_distances forms them."""
    X = np.asarray(X, dtype=np.float64)
    Y = X if Y is None else np.asarray(Y, dtype=np.float64)
    xx = np.sum(X ** 2, axis=1, keepdims=True)
    yy = np.sum(Y ** 2, axis=1, keepdims=True)
    d2 = xx - 2 * (X @ Y.T) + yy.T
    neg = d2 < 0
    d2[neg] = 0
    return np.sqrt(d2), int(neg.sum())


def radii(X, k=3):
    """(k+1)-th smallest entry of each row of the self-distance matrix (the ~0 self distance counted)."""
    d, _ = pairwise_distances(X)
    return np.partition(d, k, axis=1)[:, k]


def cover(ref, ref_radii, subj):
    """flags[j]: some reference ball holds subject j, strictly (compute_metric before its mean)."""
    d, _ = pairwise_distances(ref, subj)
    return (d < np.asarray(ref_radii)[:, None]).any(axis=0)


def realism(ref, ref_radii, subj):
    """max_i radius_i / (|ref_i - subj_j| + 1e-6) per subject, the distances as pairwise_distances forms them."""
    d, _ = pairwise_distances(ref, subj)
    return (np.asarray(ref_radii)[:, None] / (d + 1e-6)).max(axis=0)


def precision_recall(real, fake, k=3):
    r_real, r_fake = radii(real, k), radii(fake, k)
    return float(cover(real, r_real, fake).mean()), float(cover(fake, r_fake, real).mean())
