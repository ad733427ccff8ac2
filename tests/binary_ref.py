"""numpy restatements of the binary corpus shard contract (include/sgpt_b200.h, binary corpus shards): the packing, the
popcounts, the sign dot product s and s / D, and the fixed-order asymmetric rescoring score of sgpt_rerank."""
import numpy as np


def pack(x, t=None):
    """fp32 [n, D] -> uint8 [n, D / 8]: np.packbits(x > t) (t None: 0); strict, NaN -> 0."""
    x = np.asarray(x, dtype=np.float32)
    t = np.zeros(x.shape[1], np.float32) if t is None else np.asarray(t, dtype=np.float32)
    with np.errstate(invalid="ignore"):
        return np.packbits(x > t[None, :], axis=1)


def popcounts(bits):
    """uint8 [n, B] -> int32 [n]."""
    return np.unpackbits(np.asarray(bits, dtype=np.uint8), axis=1).sum(1).astype(np.int32)


def signs(bits):
    """uint8 [n, B] -> int8 [n, 8 B] of +-1 (+1 where the bit is set)."""
    return np.unpackbits(np.asarray(bits, dtype=np.uint8), axis=1).astype(np.int8) * 2 - 1


def sign_dot(qbits, dbits):
    """s = D - 2 hamming of every (query, document) pair, computed from a = popc(q AND d): 4 a - 2 pd - 2 pq + D, int64."""
    qbits, dbits = np.asarray(qbits, np.uint8), np.asarray(dbits, np.uint8)
    D = 8 * qbits.shape[1]
    a = np.unpackbits(qbits[:, None, :] & dbits[None, :, :], axis=2).sum(2).astype(np.int64)
    return 4 * a - 2 * popcounts(dbits)[None, :].astype(np.int64) - 2 * popcounts(qbits)[:, None].astype(np.int64) + D


def cos_of(s, D):
    """cos_sim of the +-1 vectors: one correctly rounded fp32 division s / D."""
    return np.asarray(s, dtype=np.float32) / np.float32(D)


def asym_scores(q, bits, q_scale=None):
    """sgpt_rerank's SGPT_DTYPE_B1 score of fp32 query rows q [m, D] against bit rows [m, D / 8] (pair i = (q[i],
    bits[i])), in the header's order: lane l sums the 128-dimension units l, l + 32, ... in ascending order, each unit's
    dimensions ascending, acc += bit ? q : -q in fp32; then the xor butterfly over the 32 lanes; then x q_scale (fp32
    [m] or None), NaN -> -1."""
    q = np.asarray(q, dtype=np.float32)
    m, D = q.shape
    sgn = signs(bits).astype(np.float32)
    acc = np.zeros((m, 32), np.float32)
    units = D // 128
    for l in range(32):
        for u in range(l, units, 32):
            for j in range(128 * u, 128 * u + 128):
                acc[:, l] = np.where(sgn[:, j] > 0, acc[:, l] + q[:, j], acc[:, l] - q[:, j]).astype(np.float32)
    for o in (16, 8, 4, 2, 1):
        acc = (acc + acc[:, np.arange(32) ^ o]).astype(np.float32)
    x = acc[:, 0]
    if q_scale is not None:
        x = (x * np.asarray(q_scale, np.float32)).astype(np.float32)
    return np.where(np.isnan(x), np.float32(-1), x).astype(np.float32)


def inv_sqrt_dim(D):
    """The cos_sim q_scale of the binary rescoring: fp32(1 / sqrt(D))."""
    return np.float32(1.0 / np.sqrt(np.float64(D)))
