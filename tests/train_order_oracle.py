"""NumPy restatement of the shuffled order of ``hr_sample_train_batch`` (csrc/hr_train_batch.cu).

Epoch ``e`` with seed ``s`` visits pixel ``order(n, s, e)[p]`` at position ``p``: a Feistel network over ``[0, 2^k)``, ``2^k``
the next power of two >= ``n``, walked in cycles until the value falls below ``n``.  The ``k`` bits split into a low half of
``k // 2`` bits and a high half of ``k - k // 2``; six rounds alternately XOR the low half with ``F(high)`` (even rounds) and the
high half with ``F(low)`` (odd rounds), ``F(v) = mix64(v ^ round_key)`` masked to the half's width, ``mix64`` the splitmix64
finaliser.  Keys: ``epoch_key = mix64(mix64(seed) + G * (epoch + 1))``, ``round_key[i] = mix64(epoch_key + G * (i + 1))``,
``G = 0x9E3779B97F4A7C15``, all modulo 2^64.
"""
import numpy as np

ROUNDS = 6
GOLDEN = 0x9E3779B97F4A7C15
M64 = (1 << 64) - 1


def mix64_int(z: int) -> int:
    z &= M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def mix64(z: np.ndarray) -> np.ndarray:
    z = z.astype(np.uint64)
    with np.errstate(over="ignore"):
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def round_keys(seed: int, epoch: int):
    epoch_key = mix64_int(mix64_int(seed) + GOLDEN * ((epoch + 1) & M64))
    return [mix64_int(epoch_key + GOLDEN * (i + 1)) for i in range(ROUNDS)]


def feistel(x: np.ndarray, n: int, keys) -> np.ndarray:
    """One pass of the network over ``[0, 2^k)`` (no cycle-walking)."""
    bits = 0
    while (1 << bits) < n:
        bits += 1
    lo_bits = bits // 2
    lo_mask, hi_mask = np.uint64((1 << lo_bits) - 1), np.uint64((1 << (bits - lo_bits)) - 1)
    x = x.astype(np.uint64)
    lo, hi = x & lo_mask, x >> np.uint64(lo_bits)
    for i, k in enumerate(keys):
        if i & 1:
            hi = hi ^ (mix64(lo ^ np.uint64(k)) & hi_mask)
        else:
            lo = lo ^ (mix64(hi ^ np.uint64(k)) & lo_mask)
    return (hi << np.uint64(lo_bits)) | lo


def permute(p: np.ndarray, n: int, seed: int, epoch: int) -> np.ndarray:
    """The pixel at positions ``p`` of the epoch's order (cycle-walking included)."""
    keys = round_keys(seed, epoch)
    x = feistel(np.asarray(p, dtype=np.uint64), n, keys)
    out = x >= np.uint64(n)
    while out.any():
        x[out] = feistel(x[out], n, keys)
        out = x >= np.uint64(n)
    return x.astype(np.int64)


def order(n: int, seed: int, epoch: int) -> np.ndarray:
    """The whole epoch: ``order[p]`` is the pixel visited at position ``p``."""
    return permute(np.arange(n, dtype=np.uint64), n, seed, epoch)
