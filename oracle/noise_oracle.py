"""The noise of fused objectives with rand() / randn() (csrc/evok_sampler.cuh: noise_bits, noise4, noise1, value_rand,
value_randn), restated in numpy on es_oracle.philox4x32_10.

Occurrence k (0 .. 3 in the element terms, 4 .. 7 in `value`, in source order) at global row `row` takes the Philox counter

    (x, row & 0xFFFFFFFF, 0x80000000 | k << 24 | (row >> 32) & 0xFFFFFF, stream word)

with x = the column group j // 4 for an element occurrence and 0xFFFFFFFF for one in `value`, on the key of the population's
draw (seed, stream id).  A sample counter (es_oracle.philox_normals) is (q, unit & 0xFFFFFFFF, unit >> 32, stream word), whose
third word is below 2^31 for every unit below 2^63, so the two never meet.
"""

from __future__ import annotations

import numpy as np

from .es_oracle import _box_muller, philox4x32_10

VALUE_X = 0xFFFFFFFF
VALUE_K0 = 4  # the first occurrence index of `value`


def _key(seed: int, stream_id: int) -> tuple:
    return seed & 0xFFFFFFFF, ((seed >> 32) ^ (stream_id >> 32)) & 0xFFFFFFFF


def noise_counter(x, row, k: int, stream_word: int) -> tuple:
    """The 4 counter words (uint64 arrays) of occurrence k at rows `row` and first words `x` (broadcast together)."""
    row = np.asarray(row, dtype=np.uint64)
    x = np.asarray(x, dtype=np.uint64)
    x, row = np.broadcast_arrays(x, row)
    c2 = np.uint64(0x80000000) | np.uint64(k << 24) | ((row >> np.uint64(32)) & np.uint64(0xFFFFFF))
    return x, row & np.uint64(0xFFFFFFFF), c2, np.full(x.shape, stream_word & 0xFFFFFFFF, dtype=np.uint64)


def sample_counter(q, unit, stream_word: int) -> tuple:
    """The counter of the sampler's normals of column group q of `unit` (es_oracle.philox_normals)."""
    unit = np.asarray(unit, dtype=np.uint64)
    q = np.asarray(q, dtype=np.uint64)
    q, unit = np.broadcast_arrays(q, unit)
    return q, unit & np.uint64(0xFFFFFFFF), unit >> np.uint64(32), np.full(q.shape, stream_word & 0xFFFFFFFF, dtype=np.uint64)


def uniform24(w) -> np.ndarray:
    """rand(): (w >> 8) * 2^-24, exact in float32 (returned as float64)."""
    return (np.asarray(w, dtype=np.uint32) >> np.uint32(8)).astype(np.float64) * 2.0**-24


def element_noise(seed: int, stream_id: int, rows, D: int, k: int, normal: bool) -> np.ndarray:
    """[len(rows), D]: element occurrence k at every column of the global rows (float64; rand() exact, randn() the Box-Muller
    of the sampler in float64, which the kernels' fast intrinsics match to ~1e-5)."""
    rows = np.asarray(rows, dtype=np.uint64)
    nq = (D + 3) // 4
    R, Q = np.meshgrid(rows, np.arange(nq, dtype=np.uint64), indexing="ij")
    x, y, z, w = philox4x32_10(*noise_counter(Q, R, k, stream_id), *_key(seed, stream_id))
    if normal:
        a, b = _box_muller(x, y)
        c, d = _box_muller(z, w)
        out = np.stack([a, b, c, d], axis=-1)
    else:
        out = np.stack([uniform24(x), uniform24(y), uniform24(z), uniform24(w)], axis=-1)
    return out.reshape(len(rows), nq * 4)[:, :D]


def value_noise(seed: int, stream_id: int, rows, k: int, normal: bool) -> np.ndarray:
    """[len(rows)]: occurrence k (VALUE_K0 .. VALUE_K0 + 3) of `value` at the global rows: rand() from word x, randn() the first
    normal of box_muller(x, y)."""
    x, y, _, _ = philox4x32_10(*noise_counter(VALUE_X, rows, k, stream_id), *_key(seed, stream_id))
    return _box_muller(x, y)[0] if normal else uniform24(x)
