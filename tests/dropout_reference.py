"""The dropout masks of the training step (DELORA_TRAIN_DROPOUT) in numpy, restated from the contract in
include/delora_b200.h (test infrastructure, imported like helpers): Philox4x32-10 and the keep rule.  It uses neither the
kernels nor dropout.cuh."""
import numpy as np

_M32 = np.uint64(0xFFFFFFFF)
KEEP_BELOW = 13421773           # 0.8f == 13421773 * 2^-24
INPUT, STAGE3, FC = 0, 1, 2     # tensor ids


def philox4x32_10(counter, key):
    """Philox4x32-10 on arrays: counter = 4 uint32 arrays (broadcastable), key = 2 uint32 -> 4 uint64 arrays."""
    c0, c1, c2, c3 = (np.asarray(c, dtype=np.uint64) & _M32 for c in counter)
    k0, k1 = np.uint64(key[0]) & _M32, np.uint64(key[1]) & _M32
    for _ in range(10):
        p0, p1 = c0 * np.uint64(0xD2511F53), c2 * np.uint64(0xCD9E8D57)
        c0, c1, c2, c3 = ((p1 >> np.uint64(32)) ^ c1 ^ k0) & _M32, p1 & _M32, ((p0 >> np.uint64(32)) ^ c3 ^ k1) & _M32, \
            p0 & _M32
        k0, k1 = (k0 + np.uint64(0x9E3779B9)) & _M32, (k1 + np.uint64(0xBB67AE85)) & _M32
    return c0, c1, c2, c3


def keep_mask(seed, step, tensor, n):
    """The numpy re-implementation of the contract in include/delora_b200.h -> bool [n]."""
    seed, step = int(seed) & 0xFFFFFFFFFFFFFFFF, int(step) & 0xFFFFFFFFFFFFFFFF
    i = np.arange(int(n), dtype=np.uint64)
    words = philox4x32_10((i >> np.uint64(2), tensor, step & 0xFFFFFFFF, step >> 32), (seed & 0xFFFFFFFF, seed >> 32))
    word = np.choose((i & np.uint64(3)).astype(np.int64), words)
    return (word >> np.uint64(8)) < np.uint64(KEEP_BELOW)
