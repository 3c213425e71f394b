"""numpy oracle of the stochastic optimiser's device work (pilco_normals, pilco_adam_update; DESIGN.md section 32):
Philox4x32-10 of the counter (j low, j high, stream, iteration) under the seed, the two uniforms of each pair, Box-Muller,
and the Adam step in the device's order of operations, the gradient norm summed over SGD_LANES lanes then a halving
tree.  Every Adam step is a product, a sum, a division or a square root rounded once, so a faithful implementation
matches it bit for bit; the normals go through log, sin and cos, which match to a few ulps."""
import numpy as np

LANES = 256
M0, M1, W0, W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
MASK = 0xFFFFFFFF


def philox(ctr, key):
    """Philox4x32-10: ctr [..., 4], key [..., 2] (uint32-valued) -> [..., 4] uint64 arrays holding uint32 values"""
    c = [np.asarray(ctr, dtype=np.uint64)[..., i] for i in range(4)]
    k0, k1 = (np.asarray(key, dtype=np.uint64)[..., i] for i in range(2))
    for r in range(10):
        if r:
            k0, k1 = (k0 + np.uint64(W0)) & np.uint64(MASK), (k1 + np.uint64(W1)) & np.uint64(MASK)
        p0, p1 = np.uint64(M0) * c[0], np.uint64(M1) * c[2]
        hi0, lo0 = p0 >> np.uint64(32), p0 & np.uint64(MASK)
        hi1, lo1 = p1 >> np.uint64(32), p1 & np.uint64(MASK)
        c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
    return np.stack(c, axis=-1)


def uniform(a, b):
    """(((a << 32 | b) >> 11) + 0.5) 2^-53, exact"""
    x = ((np.asarray(a, dtype=np.uint64) << np.uint64(32)) | np.asarray(b, dtype=np.uint64)) >> np.uint64(11)
    return (x.astype(np.float64) + 0.5) * 2.0 ** -53


def pair_uniforms(seed, stream, iteration, pairs):
    """(u1, u2) [pairs] of pairs 0 .. pairs-1"""
    j = np.arange(pairs, dtype=np.uint64)
    ctr = np.stack([j & np.uint64(MASK), j >> np.uint64(32), np.full_like(j, stream & MASK),
                    np.full_like(j, iteration & MASK)], axis=-1)
    key = np.array([seed & MASK, (seed >> 32) & MASK], dtype=np.uint64)
    x = philox(ctr, np.broadcast_to(key, (pairs, 2)))
    return uniform(x[:, 0], x[:, 1]), uniform(x[:, 2], x[:, 3])


def sincospi(x):
    """(sin(pi x), cos(pi x)) for x in [0, 2), the argument reduced exactly to [0, 1/4] first"""
    x = np.asarray(x, dtype=np.float64)
    ss = np.where(x >= 1.0, -1.0, 1.0)
    cs = ss.copy()
    x = np.where(x >= 1.0, x - 1.0, x)
    cs = np.where(x > 0.5, -cs, cs)
    x = np.where(x > 0.5, 1.0 - x, x)
    swap = x > 0.25
    x = np.where(swap, 0.5 - x, x)
    a, b = np.sin(np.pi * x), np.cos(np.pi * x)
    return ss * np.where(swap, b, a), cs * np.where(swap, a, b)


def normals(seed, stream, iteration, n):
    """the n normals of pilco_normals(seed, stream, *iter = iteration)"""
    u1, u2 = pair_uniforms(int(seed) % 2 ** 64, int(stream), int(iteration), (n + 1) // 2)
    r = np.sqrt(-2.0 * np.log(u1))
    s, c = sincospi(2.0 * u2)
    return np.stack([r * c, r * s], axis=-1).reshape(-1)[:n]


def sumsq(g):
    """sum g^2 in the device's order: lane l sums g[l], g[l + 256], ... in order, then s[l] += s[l + h] for
    h = 128, 64, ..., 1"""
    g = np.asarray(g, dtype=np.float64)
    n = g.shape[0]
    pad = np.zeros(-(-n // LANES) * LANES)
    pad[:n] = g
    s = np.zeros(LANES)
    for row in pad.reshape(-1, LANES):
        s = s + row * row
    h = LANES // 2
    while h:
        s[:h] = s[:h] + s[h:2 * h]
        h //= 2
    return s[0]


def adam(theta, packed, m, v, t, b1t, b2t, k, trace, ok, lr, b1, b2, eps, max_norm):
    """one pilco_adam_update on copies -> dict(theta, m, v, t, b1t, b2t, trace, ok, iter=k + 1); packed [R, n + 2]"""
    theta, m, v = theta.copy(), m.copy(), v.copy()
    t, b1t, b2t, trace, ok = t.copy(), b1t.copy(), b2t.copy(), trace.copy(), ok.copy()
    R, n = theta.shape
    for r in range(R):
        loss, status, g = packed[r, 0], packed[r, 1], packed[r, 2:2 + n].copy()
        good = status == 0.0 and np.isfinite(loss) and np.isfinite(g).all()
        if good:
            norm = np.sqrt(sumsq(g))
            if max_norm > 0.0 and norm > max_norm:
                g = g * (max_norm / norm)
            t[r] += 1
            b1t[r], b2t[r] = b1t[r] * b1, b2t[r] * b2
            m[r] = b1 * m[r] + (1.0 - b1) * g
            v[r] = b2 * v[r] + (1.0 - b2) * (g * g)
            mh, vh = m[r] / (1.0 - b1t[r]), v[r] / (1.0 - b2t[r])
            theta[r] = theta[r] - (lr * mh) / (np.sqrt(vh) + eps)
        if 0 <= k < trace.shape[0]:
            trace[k, r], ok[k, r] = -loss, good
    return dict(theta=theta, m=m, v=v, t=t, b1t=b1t, b2t=b2t, trace=trace, ok=ok, iter=k + 1)
