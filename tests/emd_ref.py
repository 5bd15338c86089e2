"""numpy restatement of genre_b200_emd_forward (include/genre_b200.h), bit for bit: the Jacobi auction with eps-scaling, its
tie rules, the effective-eps floor, the refusal and round cap, and the halving sum of the matched costs.  Plus the gradient
formula of postprocess.emd and the exact optimum by scipy's linear_sum_assignment on the same costs."""
import numpy as np

MAX_ROUNDS = 1 << 22
COORD_MAX = np.float32(2.0 ** 62)


def costs(p, q):
    """c_ij = sqrt((dx*dx + dy*dy) + dz*dz) in fp32, d = p_i - q_j, one rounding per operation (numpy never fuses)"""
    p, q = np.asarray(p, np.float32), np.asarray(q, np.float32)
    d = p[:, None, :] - q[None, :, :]
    s = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
    return np.sqrt(s)


def eps_schedule(p, q, eps):
    """(D, eps_eff, eps_0) of one pair"""
    both = np.concatenate([np.asarray(p, np.float32), np.asarray(q, np.float32)])
    e = both.max(0).astype(np.float64) - both.min(0).astype(np.float64)
    D = np.sqrt((e[0] * e[0] + e[1] * e[1]) + e[2] * e[2])
    eps_eff = max(float(eps), float(np.ldexp(D, -32)))
    return float(D), eps_eff, max(float(D * 0.25), eps_eff)


def refused(p, q):
    both = np.concatenate([np.asarray(p, np.float32), np.asarray(q, np.float32)])
    return not (np.abs(both) <= COORD_MAX).all()


def halving_sum(a):
    """zero-pad to a power of two and add the upper half onto the lower one until one value is left"""
    n2 = 1
    while n2 < len(a):
        n2 *= 2
    a = np.concatenate([np.asarray(a, np.float64), np.zeros(n2 - len(a))])
    while len(a) > 1:
        h = len(a) // 2
        a = a[:h] + a[h:]
    return a[0]


def auction(p, q, eps, max_rounds=MAX_ROUNDS):
    """one pair -> (match [n] int32, emd fp64, rounds, phases, eps_eff)"""
    n = len(p)
    if refused(p, q):
        return np.full(n, -1, np.int32), np.nan, 0, 0, np.nan
    C = costs(p, q).astype(np.float64)
    _, eps_eff, eps_k = eps_schedule(p, q, eps)
    price = np.zeros(n)
    rounds = phases = 0
    while True:
        phases += 1
        assign = np.full(n, -1, np.int64)
        owner = np.full(n, -1, np.int64)
        bidders = np.arange(n)
        while True:
            rounds += 1
            V = np.negative(C[bidders]) - price[None, :]
            r = np.arange(len(bidders))
            j1 = V.argmax(1)                                   # the first (lowest) j of the maximum
            v1 = V[r, j1]
            if n > 1:
                V[r, j1] = -np.inf
                v2 = V.max(1)
            else:
                v2 = v1
            bid = (price[j1] + (v1 - v2)) + eps_k
            order = np.lexsort((bidders, -bid, j1))            # per object: the highest bid, then the lowest bidder
            first = np.ones(len(order), bool)
            first[1:] = j1[order][1:] != j1[order][:-1]
            win = order[first]
            wj, wi = j1[win], bidders[win]
            old = owner[wj]
            assign[old[old >= 0]] = -1
            owner[wj] = wi
            assign[wi] = wj
            price[wj] = bid[win]
            bidders = np.nonzero(assign < 0)[0]
            if len(bidders) == 0:
                break
            if rounds >= max_rounds:
                return np.full(n, -1, np.int32), np.nan, rounds, phases, eps_eff
        if eps_k == eps_eff:
            break
        eps_k = max(eps_k * 0.25, eps_eff)
    matched = C[np.arange(n), assign]
    s = matched[0] if n == 1 else halving_sum(matched)
    return assign.astype(np.int32), s / n, rounds, phases, eps_eff


def emd(p, q, eps):
    """batches [B, n, 3] -> (emd [B] fp64, match [B, n] int32, rounds [B], phases [B])"""
    out = [auction(a, b, eps) for a, b in zip(p, q)]
    return (np.array([o[1] for o in out]), np.stack([o[0] for o in out]), np.array([o[2] for o in out]),
            np.array([o[3] for o in out]))


def optimum(p, q):
    """the exact optimal mean cost of one pair on the same fp32 costs, widened to fp64"""
    from scipy.optimize import linear_sum_assignment
    C = costs(p, q).astype(np.float64)
    r, c = linear_sum_assignment(C)
    return C[r, c].mean()


def grad(p, q, match):
    """dEMD/dp and dEMD/dq of one pair at a fixed matching, fp64: (p_i - q_s(i)) / (n c_i), 0 where c_i = 0"""
    p, q = np.asarray(p, np.float64), np.asarray(q, np.float64)
    n = len(p)
    d = p - q[match]
    c = np.sqrt((d * d).sum(1))
    gp = np.where(c[:, None] > 0, d / (n * np.where(c > 0, c, 1.0))[:, None], 0.0)
    gq = np.zeros_like(q)
    gq[match] = -gp
    return gp, gq
