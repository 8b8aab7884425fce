"""numpy restatement of include/gpd_b200_sis.h: Philox4x32-10 and the draws of one SIS round of one cloud.

The parent and uniform-point choices are integer arithmetic and match the library exactly; the Gaussian offsets use numpy's
log / cos / sin (the library: log, cospi, sinpi), so positions agree to ~1e-15 relative, not bit for bit.
"""
import numpy as np

MAX_PROPOSALS = 1 << 20
M0, M1, W0, W1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57), np.uint32(0x9E3779B9), np.uint32(0xBB67AE85)
MASK = np.uint64(0xFFFFFFFF)


def philox(ctr, key):
    """Philox4x32-10 of counters ctr [n, 4] (uint32) under key (k0, k1) -> [n, 4] uint32."""
    c = [np.asarray(ctr, np.uint32)[:, i].astype(np.uint64) for i in range(4)]
    k0, k1 = np.uint32(key[0]), np.uint32(key[1])
    for _ in range(10):
        p0, p1 = M0 * c[0], M1 * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ np.uint64(k0), p1 & MASK, (p0 >> np.uint64(32)) ^ c[3] ^ np.uint64(k1), p0 & MASK]
        k0, k1 = np.uint32((int(k0) + int(W0)) & 0xFFFFFFFF), np.uint32((int(k1) + int(W1)) & 0xFFFFFFFF)
    return np.stack(c, axis=1).astype(np.uint32)


def draws(key, t, r, stream, half):
    """The draws of proposals t (array) of round r: key = seed + b (uint64)."""
    t = np.asarray(t, np.uint32)
    ctr = np.stack([t, np.full_like(t, r), np.full_like(t, stream), np.full_like(t, half)], axis=1)
    return philox(ctr, (int(key) & 0xFFFFFFFF, int(key) >> 32))


def unit(w):
    return (w.astype(np.float64) + 0.5) * 2.0 ** -32


def gaussian(key, t, r, m):
    """(parent index, z [n, 3]) of Gaussian proposals t."""
    c0, c1 = draws(key, t, r, 0, 0), draws(key, t, r, 0, 1)
    r01, a01 = np.sqrt(-2.0 * np.log(unit(c0[:, 1]))), 2.0 * unit(c0[:, 2])
    z = np.stack([r01 * np.cos(np.pi * a01), r01 * np.sin(np.pi * a01),
                  np.sqrt(-2.0 * np.log(unit(c0[:, 3]))) * np.cos(np.pi * 2.0 * unit(c1[:, 0]))], axis=1)
    return (c0[:, 0] % np.uint32(m)).astype(np.int64), z


def d2(x, k):
    d = x - k
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def draw_round(kept, r, key, S, prob_rand, sigma, method, workspace, xyz, init, wave=4096):
    """The positions of round r of one cloud with kept positions kept [m, 3] (m > 0), its points xyz [N, 3] float32 and
    initial indices init. Returns (positions [n, 3], parents [n_gauss accepted], n_gauss accepted)."""
    n_rand = int(prob_rand * S)
    n_gauss = S - n_rand
    m = len(kept)
    out, parents = [], []
    t0 = 0
    while len(out) < n_gauss and t0 < MAX_PROPOSALS:
        t = np.arange(t0, min(t0 + wave, MAX_PROPOSALS))
        par, z = gaussian(key, t, r, m)
        x = kept[par] + sigma * z
        acc = np.ones(len(t), bool)
        if method == 1:
            acc = d2(x, kept[par]) <= d2(x[:, None, :], kept[None, :, :]).min(axis=1)
        for i in np.flatnonzero(acc)[: n_gauss - len(out)]:
            out.append(x[i])
            parents.append(par[i])
        t0 += wave
    ng = len(out)
    ws = np.asarray(workspace, np.float64)
    t0, nr = 0, 0
    while nr < n_rand and t0 < MAX_PROPOSALS:
        t = np.arange(t0, min(t0 + wave, MAX_PROPOSALS))
        c = draws(key, t, r, 1, 0)[:, 0]
        pi = np.asarray(init)[c % np.uint32(len(init))] if len(init) else (c % np.uint32(len(xyz))).astype(np.int64)
        p = xyz[pi].astype(np.float64)
        acc = np.all((p >= ws[0::2]) & (p <= ws[1::2]), axis=1)
        for i in np.flatnonzero(acc)[: n_rand - nr]:
            out.append(p[i])
            nr += 1
        t0 += wave
    return np.array(out, np.float64).reshape(-1, 3), np.array(parents, np.int64), ng
