"""Synthetic descriptor sets for the large-capacity texture matchers (k_texture_knn_hamming / k_texture_knn_l2), made
from a fixed integer hash rather than stored: tests/golden/texture_knn_large.npz keeps only cv2.BFMatcher's kNN results
for them. Every set has pinned cases around the matchers' 512-row train chunks:

- rows n - 513 and n - 1 are equal (n > 512); one query equals them (distance 0 to both: the ratio test's 0 / 0 keeps
  the match, and the earlier row must win across the chunk boundary), another sits at the same non-zero distance from
  both (ratio 1 drops it);
- rows 3, 10, 17, ... are at the same distance from the zero query, the last query (the first two marked rows are its
  neighbours, ratio 1); every other row is farther from it;
- 24 random queries.

Rows are uint8: 32 bytes for Hamming, 128 whole numbers in 0 .. 63 for L2 (exact in float in any summation order)."""
import numpy as np

SIZES = (511, 512, 513, 1024, 4096)
_GOLDEN = np.uint64(0x9E3779B97F4A7C15)


def _bytes(seed, shape):
    """splitmix64 of 1, 2, ... offset by `seed`, as uint8: the same on every platform and NumPy version."""
    n = int(np.prod(shape))
    x = np.arange(1, (n + 7) // 8 + 1, dtype=np.uint64) * _GOLDEN + np.uint64(seed)
    x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    x = x ^ (x >> np.uint64(31))
    return x.astype("<u8").view(np.uint8)[:n].reshape(shape)


def synthetic(n, hamming):
    """(queries, train) as uint8 rows for a train set of n rows."""
    width = 32 if hamming else 128
    seed = n * 2 + (1 if hamming else 0)
    t = _bytes(seed * 1000003, (n, width))
    q = list(_bytes(seed * 1000003 + 7919, (24, width)))
    if not hamming:  # L2 rows in 0 .. 63 stay far apart from each other
        t = t & np.uint8(63)
        q = [r & np.uint8(63) for r in q]
    for j in range(n):
        if j % 7 == 3:
            t[j] = 0
            if hamming:
                t[j, j % 32] = 1 << (j // 32 % 8)  # distance 1 from the zero query
            else:
                t[j, j % 128] = 10  # distance 10
        elif hamming:
            t[j, :2] |= 0x0F  # at least 8 bits from the zero query
        else:
            t[j, 0] = max(t[j, 0], 40)  # at least 40 from it
    if n > 512:  # neither n - 513 nor n - 1 is a marked row for the sizes above
        t[n - 513] = t[n - 1]
        q.append(t[n - 1].copy())
        near = t[n - 1].copy()
        if hamming:
            near[3] ^= 1
        else:
            near[3] += 1
        q.append(near)
    q.append(np.zeros(width, np.uint8))
    return np.stack(q), t
