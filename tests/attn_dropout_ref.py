"""numpy replica of the attention-dropout keep mask (include/magvit2_b200.h, mv2_dropout_args): Philox4x32-10 and the keep rule,
written from the published algorithm (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC'11; Random123's round
constants), independent of the CUDA code it checks."""
import numpy as np

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)
LO = np.uint64(0xFFFFFFFF)
S32 = np.uint64(32)


def philox4x32_10(ctr, key):
    """ctr (..., 4) and key (..., 2) uint32 arrays (broadcast) -> (..., 4) uint32."""
    c = [np.asarray(ctr[..., n], dtype=np.uint64) for n in range(4)]
    k0 = np.asarray(key[..., 0], dtype=np.uint64)
    k1 = np.asarray(key[..., 1], dtype=np.uint64)
    for r in range(10):
        if r:
            k0, k1 = (k0 + W0) & LO, (k1 + W1) & LO
        p0, p1 = M0 * c[0], M1 * c[2]               # 32 x 32 -> 64 bit, exact in uint64
        c = [(p1 >> S32) ^ c[1] ^ k0, p1 & LO, (p0 >> S32) ^ c[3] ^ k1, p0 & LO]
    return np.stack(c, axis=-1).astype(np.uint32)


def keep_threshold(p):
    """floor(p * 2^32) of the fp32 value of p: a word is kept iff it is >= this."""
    return int(np.floor(float(np.float32(p)) * 2.0 ** 32))


def dropout_scale(p):
    """fp32(1 / (1 - p)) of the fp32 value of p."""
    return float(np.float32(1.0 / (1.0 - float(np.float32(p)))))


def keep_mask(seed, call, p, n_seq, heads, L, n_mem):
    """uint8 keep[seq][h][i][n_mem + L]: word j & 3 of philox((i, j >> 2, seq, h | call << 16), (seed lo, seed hi))."""
    M = n_mem + L
    G = (M + 3) // 4
    s, h, i, g = np.meshgrid(np.arange(n_seq, dtype=np.uint32), np.arange(heads, dtype=np.uint32),
                             np.arange(L, dtype=np.uint32), np.arange(G, dtype=np.uint32), indexing="ij")
    ctr = np.stack((i, g, s, h | np.uint32(call << 16)), axis=-1)
    key = np.array([seed & 0xFFFFFFFF, seed >> 32], dtype=np.uint32)
    words = philox4x32_10(ctr, key).reshape(n_seq, heads, L, 4 * G)[..., :M]
    return (words >= np.uint32(keep_threshold(p))).astype(np.uint8)          # 0 < p < 1: the threshold is below 2^32
