"""TEST ORACLE: the RNG contract of seeded sampling (ts_pixelcnn_sample_seeded, include/talkshow_b200.h) in numpy.

Philox4x32-10 (the Random123 / cuRAND counter-based generator) in uint64 arithmetic, vectorised over counters, and the
builder of the [2T,B,2048] noise tensor the seeded sampler divides by.  Draw (absolute row r, column c, code n) of a clip
with seed s uses output n >> 9 of counter (n & 511, r, c, 0) under key (s & 0xffffffff, s >> 32); u = ((x >> 8) | 1) 2^-24,
q = -log(u)."""
import numpy as np

M0, M1 = 0xD2511F53, 0xCD9E8D57          # round multipliers
W0, W1 = 0x9E3779B9, 0xBB67AE85          # key increments (Weyl sequence)
MASK = 0xFFFFFFFF


def philox4x32_10(ctr, key):
    """ctr [..., 4], key [..., 2] (broadcastable, integers < 2^32) -> [..., 4] uint32."""
    c = [np.asarray(ctr, dtype=np.uint64)[..., i] for i in range(4)]
    k0, k1 = (np.asarray(key, dtype=np.uint64)[..., i] for i in range(2))
    for _ in range(10):
        p0 = np.uint64(M0) * c[0]
        p1 = np.uint64(M1) * c[2]
        hi0, lo0 = p0 >> np.uint64(32), p0 & np.uint64(MASK)
        hi1, lo1 = p1 >> np.uint64(32), p1 & np.uint64(MASK)
        c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
        k0 = (k0 + np.uint64(W0)) & np.uint64(MASK)
        k1 = (k1 + np.uint64(W1)) & np.uint64(MASK)
    return np.stack(c, -1).astype(np.uint32)


def seed_key(seed):
    """int64 seed (any integer, taken as its low 64 bits) -> key (lo, hi)."""
    s = int(seed) & 0xFFFFFFFFFFFFFFFF
    return s & MASK, s >> 32


def uniforms_block(seeds, T, T0=0):
    """u [2T,B,2048] float64 (every value exact in fp32): block 2(r-T0)+c holds draw (r, c) for rows r in [T0, T0+T)."""
    keys = np.array([seed_key(s) for s in np.asarray(seeds, dtype=object).reshape(-1)], dtype=np.uint64)   # [B,2]
    B = keys.shape[0]
    shape = (T, 2, B, 512)
    ctr = np.stack([np.broadcast_to(np.arange(512), shape), np.broadcast_to((T0 + np.arange(T))[:, None, None, None], shape),
                    np.broadcast_to(np.arange(2)[None, :, None, None], shape), np.zeros(shape, dtype=np.int64)], -1)
    x = philox4x32_10(ctr, keys[None, None, :, None, :])                  # [T,2,B,512,4]: counter m, output j
    x = x.swapaxes(-1, -2).reshape(2 * T, B, 2048).astype(np.uint64)      # code n = 512 j + m
    return ((x >> np.uint64(8)) | np.uint64(1)).astype(np.float64) * 2.0 ** -24


def uniforms(seed, r, c):
    """u [2048] of draw (r, c) of the clip seeded `seed`."""
    return uniforms_block([seed], 1, r)[c, 0]


def noise(seeds, T, T0=0):
    """The seeded sampler's q as float32 [2T,B,2048]: -log(u) in float64, rounded once to fp32 (the device's logf is
    within one ulp of it)."""
    return (-np.log(uniforms_block(seeds, T, T0))).astype(np.float32)
