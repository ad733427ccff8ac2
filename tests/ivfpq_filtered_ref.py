"""numpy restatement of the filtered IVF-PQ search (include/sgpt_b200.h, sgpt_ivfpq_search_masked).

Top-k over each query's probed positions that its bitmap allows and whose doc_ids entry is >= 0, by ADC score
(sum_j lut[q][j][code_j] + base[q][p] for the probe p covering the position), score descending, ties by ascending global
id, tail (-inf, -1).  The sums are taken in fp64: with integer-valued tables they are exact, and so equal to the device's
fp32 sums in any order."""
import numpy as np


def unpack_codes(codes: np.ndarray, nbits: int) -> np.ndarray:
    """Stored code rows uint8 [n, m nbits / 8] -> codes int64 [n, m] (4-bit: the even subspace in the low nibble)."""
    codes = codes.astype(np.int64)
    if nbits == 8:
        return codes
    out = np.empty((codes.shape[0], 2 * codes.shape[1]), dtype=np.int64)
    out[:, 0::2], out[:, 1::2] = codes & 15, codes >> 4
    return out


def adc_scores(lut: np.ndarray, base: np.ndarray, codes: np.ndarray, nbits: int, offsets: np.ndarray,
               probes: np.ndarray) -> np.ndarray:
    """[nq, n] fp64: the ADC score of every position a probe of the query covers, NaN elsewhere.  Probes outside
    [0, nlist) are skipped."""
    c = unpack_codes(codes, nbits)
    nq, m, K = lut.shape
    n, nlist = c.shape[0], offsets.size - 1
    flat = c + (np.arange(m) * K)[None, :]  # index into lut[q].reshape(-1)
    out = np.full((nq, n), np.nan)
    for q in range(nq):
        table = lut[q].reshape(-1).astype(np.float64)
        for p, l in enumerate(probes[q].tolist()):
            if 0 <= l < nlist:
                b, e = int(offsets[l]), int(offsets[l + 1])
                out[q, b:e] = table[flat[b:e]].sum(axis=1) + float(base[q, p])
    return out


def allowed(mask: np.ndarray, pitch: int, nq: int, n: int) -> np.ndarray:
    """bool [nq, n] of the bitmap argument: None (every position), one shared bitmap (pitch 0) or rows of `pitch`
    words (uint32 or int32 words, flat or [nq, pitch]); bits at or past n are never read."""
    if mask is None:
        return np.ones((nq, n), dtype=bool)
    w = np.ascontiguousarray(mask).view(np.uint32).reshape(-1)
    pos = np.arange(n)
    out = np.zeros((nq, n), dtype=bool)
    for q in range(nq):
        row = w[q * pitch:]  # pitch 0: every query reads the shared bitmap
        out[q] = (row[pos >> 5] >> (pos & 31).astype(np.uint32)) & 1
    return out


def search(scores: np.ndarray, ids: np.ndarray, allow: np.ndarray, k: int):
    """(scores fp32 [nq, k], ids int64 [nq, k]): per query the top-k of the positions with a score (probed) that
    `allow` [nq, n] allows and whose id is >= 0, score descending, ties by ascending id, tail (-inf, -1)."""
    nq = scores.shape[0]
    out_s = np.full((nq, k), -np.inf, dtype=np.float32)
    out_i = np.full((nq, k), -1, dtype=np.int64)
    ids = ids.astype(np.int64)
    for q in range(nq):
        keep = ~np.isnan(scores[q]) & allow[q] & (ids >= 0)
        s, g = scores[q][keep], ids[keep]
        order = np.lexsort((g, -s))[:k]
        out_s[q, :order.size] = s[order]
        out_i[q, :order.size] = g[order]
    return out_s, out_i
