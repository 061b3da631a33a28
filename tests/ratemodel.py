"""numpy restatement of the encoder's rate control (openjph_b200/csrc/rate_ctrl.cu): distortion tables, the per-block
lower convex hull with its slope keys, and the threshold selection.  Test infrastructure only."""
import numpy as np

INVALID = 0xFFFFFFFF


def distortion(words, K, irv):
    """unweighted sum_i (m_i - r_k(m_i))^2 for k = 0..K; words: a block's sign-magnitude words, K = K_max"""
    m = (np.asarray(words, np.uint64).ravel() & np.uint64(0x7FFFFFFF)) >> np.uint64(31 - K)
    m = m.astype(np.int64)
    D = np.zeros(K + 1)
    for k in range(K + 1):
        h = (0.5 if irv else 0.0) if k == 0 else float(1 << (k - 1))
        e = np.where((m >> k) != 0, (m & ((1 << k) - 1)).astype(np.float64) - h, m.astype(np.float64))
        D[k] = float(np.sum(e * e))
    return D


def hull(R, D, K):
    """gift wrapping from the excluded point (0, D[K]), as rc_hull_kernel: returns (ks, keys, lens), ks[0] = K,
    segment j goes from point ks[j] to ks[j + 1] with length lens[j] and key keys[j]"""
    cur_r, cur_d, last = 0, float(D[K]), INVALID
    ks, keys, lens = [K], [], []
    while True:
        best, best_s, best_r = -1, 0.0, 0
        for k in range(K):
            r = int(R[k])
            if r == INVALID or r <= cur_r or not (D[k] < cur_d):
                continue
            s = (cur_d - float(D[k])) / float(r - cur_r)
            if best < 0 or s > best_s or (s == best_s and r > best_r):
                best, best_s, best_r = k, s, r
        if best < 0:
            break
        key = min(int(np.float32(best_s).view(np.uint32)), last)
        last = key
        ks.append(best); keys.append(key); lens.append(best_r)
        cur_r, cur_d = best_r, float(D[best])
    return ks, keys, lens


def taken(keys, t):
    j = 0
    while j < len(keys) and keys[j] >= t:
        j += 1
    return j


def select(hulls, budget):
    """smallest key t with sum_b R_b(k_b(t)) <= budget (bisection over 33 bits); returns (k per block, body, t)"""
    def body(t):
        return sum(h[2][taken(h[1], t) - 1] if taken(h[1], t) else 0 for h in hulls)
    lo, hi = 0, 1 << 32
    if body(0) <= budget:
        hi = 0
    else:
        while hi - lo > 1:
            mid = (lo + hi) >> 1
            if body(mid) <= budget:
                hi = mid
            else:
                lo = mid
    ks = [h[0][taken(h[1], hi)] for h in hulls]
    return ks, body(hi), hi


def next_increment(hulls, t):
    """length increment of the highest-key hull segment not taken at threshold t (0 if every segment is taken)"""
    best_key, inc = -1, 0
    for ks, keys, lens in hulls:
        j = taken(keys, t)
        if j < len(keys) and keys[j] > best_key:
            best_key, inc = keys[j], lens[j] - (lens[j - 1] if j else 0)
    return inc
