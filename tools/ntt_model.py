"""CPU model of era_boojum_b200/csrc/ntt.cu (planner + ntt_pass_kernel index logic), transcribed statement by
statement so the tile / stage / twiddle-index arithmetic can be validated against the oracle without a GPU.
Dev tool; used by tests/test_ntt_model.py (CPU).  Not part of the product path.
"""
import numpy as np

P = 0xFFFFFFFF00000001


def brev(x, bits):
    r = 0
    for _ in range(bits):
        r = (r << 1) | (x & 1)
        x >>= 1
    return r


def omega(log_n):
    w = 0x185629DCDA58878C
    for _ in range(log_n, 32):
        w = w * w % P
    return w


def twiddle_table(log_n, inverse):
    w = omega(log_n)
    if inverse:
        w = pow(w, P - 2, P)
    bits = log_n - 1
    return [pow(w, brev(k, bits), P) for k in range(1 << bits)] if log_n >= 1 else [1]


def twist_table(log_n, coset):
    """ntt.cu get_twist_table: tw[2^r + G] = tab[G] * coset^(2^(log_n - r - 1)), r < log_n, G < 2^r (tw[0] unused)."""
    tab = twiddle_table(log_n, False)
    tw = [0] * (1 << log_n)
    for r in range(log_n):
        c = pow(coset, 1 << (log_n - r - 1), P)
        for g in range(1 << r):
            tw[(1 << r) + g] = tab[g] * c % P
    return tw


NTT_MAX_PASSES = 6  # capacity of ntt.cu's Plan


def make_plan(m, transpose_last, MAXE=13, pass1_w=-1):
    if m <= 12:
        return [(m, 0)]
    TL = MAXE - 2 if transpose_last else MAXE
    TM = MAXE - 2
    t_last = min(TL, max((m + 1) // 2, m - 10))
    rest = m - t_last
    n_front = (rest + TM - 1) // TM
    if n_front + 1 > NTT_MAX_PASSES:
        raise ValueError("plan of 2^%d (MAXE %d) needs %d passes" % (m, MAXE, n_front + 1))
    plan, r0 = [], 0
    for i in range(n_front):
        ti = rest // (n_front - i)
        rest -= ti
        wi = pass1_w if pass1_w >= 0 else max(2, min(5, MAXE - ti))
        wi = min(wi, MAXE - ti)
        wi = min(wi, m - r0 - ti)
        if ti + wi < 4:
            wi = 4 - ti
        plan.append((ti, wi))
        r0 += ti
    plan.append((t_last, min(min(MAXE - t_last, 5), r0) if transpose_last else 0))
    return plan


def run_pass(src, m, r0, t, w, kind, tab, scale=None, scale_on_load=True, twisted=False):
    """kind 0 = PASS_TILE, 1 = PASS_TRANSPOSE_LAST.  scale: function(index) -> factor or None.  twisted (PASS_TILE): tab
    is a twist_table, round rho's twiddles start at tab[2^rho]."""
    LOG_E = t + w
    E, W = 1 << LOG_E, 1 << w
    dst = [None] * (1 << m)
    n_tiles = (1 << (m - t - w)) if kind == 0 else (1 << (r0 - w))
    for tile in range(n_tiles):
        sm = [0] * E
        hi = 0
        if kind == 0:
            lo_bits = m - r0 - t
            groups_log = lo_bits - w
            S = 1 << lo_bits
            hi = tile >> groups_log
            lo0 = (tile & ((1 << groups_log) - 1)) << w
            base = (hi << (m - r0)) + lo0
            for e in range(E):
                row, col = e >> w, e & (W - 1)
                gi = base + row * S + col
                v = src[gi]
                if scale and scale_on_load:
                    v = v * scale(gi) % P
                sm[e] = v
        else:
            for idx in range(E):
                col, row = idx >> t, idx & ((1 << t) - 1)
                k1 = (tile << w) + col
                blk = brev(k1, r0) if r0 else 0
                gi = (blk << t) + row
                v = src[gi]
                if scale and scale_on_load:
                    v = v * scale(gi) % P
                sm[row * W + col] = v
        done = 0
        rs = t & 3
        if rs == 0:
            rs = 4
        nvt = E >> 4
        while done < t:
            b_lo = t - done - rs
            pp = b_lo + w - (4 - rs)
            assert pp >= 0
            for q in range(nvt):
                e0 = ((q >> pp) << (pp + 4)) | (q & ((1 << pp) - 1))
                hq = (hi | (1 << r0)) if twisted else hi
                if kind != 0:
                    k1 = (tile << w) + (e0 & (W - 1))
                    hq = brev(k1, r0) if r0 else 0
                pfx = (hq << (LOG_E - pp - 4)) | (q >> pp)
                x = [sm[e0 | (j << pp)] for j in range(16)]
                for qq in range(rs):
                    bit = 1 << (3 - qq)
                    for j0 in range(16):
                        if j0 & bit:
                            continue
                        j1 = j0 | bit
                        k = (pfx << qq) | (j0 >> (4 - qq))
                        s = tab[k]
                        v = x[j1] * s % P
                        x[j1] = (x[j0] - v) % P
                        x[j0] = (x[j0] + v) % P
                for j in range(16):
                    sm[e0 | (j << pp)] = x[j]
            done += rs
            rs = 4
        if kind == 0:
            for e in range(E):
                row, col = e >> w, e & (W - 1)
                gi = base + row * S + col
                v = sm[e]
                if scale and not scale_on_load:
                    v = v * scale(gi) % P
                dst[gi] = v
        else:
            for idx in range(E):
                col = idx & (W - 1)
                kappa = idx >> w
                rho = brev(kappa, t) if t else 0
                v = sm[rho * W + col]
                k1 = (tile << w) + col
                go = k1 + (kappa << r0)
                if scale and not scale_on_load:
                    v = v * scale(go) % P
                dst[go] = v
    assert all(v is not None for v in dst)
    return dst


def transform(a, coset=1, inverse=False, MAXE=13, pass1_w=-1, twist=False):
    """twist (forward, coset != 1): the coset folded into the twiddles (twist_table), no scaling."""
    a = [int(x) % P for x in a]
    m = len(a).bit_length() - 1
    assert m >= 4
    twisted = twist and not inverse and coset != 1
    tab = twist_table(m, coset) if twisted else twiddle_table(m, inverse)
    plan = make_plan(m, inverse, MAXE, pass1_w)
    if not inverse:
        scale = (lambda i: pow(coset, i, P)) if coset != 1 and not twisted else None
    else:
        n_inv = pow(1 << m, P - 2, P)
        cinv = pow(coset, P - 2, P)
        scale = lambda i: n_inv * pow(cinv, i, P) % P
    cur, r0 = a, 0
    for i, (t, w) in enumerate(plan):
        first, last = i == 0, i == len(plan) - 1
        kind = 1 if (inverse and last) else 0
        sc, on_load = None, True
        if not inverse and first:
            sc, on_load = scale, True
        if inverse and last:
            sc, on_load = scale, False
        cur = run_pass(cur, m, r0, t, w, kind, tab, sc, on_load, twisted)
        r0 += t
    return np.array(cur, dtype=np.uint64), plan
