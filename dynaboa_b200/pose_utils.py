"""Evaluation metrics used by the driver (reference utils/pose_utils.py:9-64): Procrustes-aligned
error.  Host-side numpy, as in the reference: PA-MPJPE is the parity metric, not a kernel target
(SURVEY.md §2).  The driver itself evaluates on the device (`Adaptor.eval_metrics` -> `dboa_eval_metrics_active`, SURVEY §8f N1);
these numpy functions remain for API compatibility (`utils.pose_utils` of the drop-in tree)."""
import numpy as np


def compute_similarity_transform(S1, S2):
    """Similarity transform (scale, rotation, translation) taking S1 closest to S2; both (N,3) or (3,N)."""
    flip = S1.shape[0] != 3 and S1.shape[0] != 2
    A, B = (S1.T, S2.T) if flip else (S1, S2)
    assert B.shape[1] == A.shape[1]
    muA, muB = A.mean(axis=1, keepdims=True), B.mean(axis=1, keepdims=True)
    A0, B0 = A - muA, B - muB
    varA = np.sum(A0 ** 2)
    K = A0.dot(B0.T)
    U, _, Vh = np.linalg.svd(K)
    V = Vh.T
    Z = np.eye(U.shape[0])
    Z[-1, -1] *= np.sign(np.linalg.det(U.dot(V.T)))
    R = V.dot(Z.dot(U.T))
    scale = np.trace(R.dot(K)) / varA
    t = muB - scale * (R.dot(muA))
    out = scale * R.dot(A) + t
    return out.T if flip else out


def compute_similarity_transform_batch(S1, S2):
    out = np.zeros_like(S1)
    for i in range(S1.shape[0]):
        out[i] = compute_similarity_transform(S1[i], S2[i])
    return out
