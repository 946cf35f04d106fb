"""An independent restatement of the reference's randn() stream (matlabfunctions.cpp:237-264), for the known-answer
tests of the library's parallel generator.  It shares nothing with the library's jump tables: xorshift128 is written
out from Marsaglia's definition, and a jump of `d` draws applies the 128 x 128 GF(2) one-step matrix raised to 12 d
by square-and-multiply in numpy.

One draw is 12 xorshift128 steps; its raw value is the 32-bit sum of (w >> 4) over those steps, and randn() returns
sum / 2^28 - 6."""
import functools

import numpy as np

SEED = (123456789, 362436069, 521288629, 88675123)     # (x, y, z, w) after randn_reseed()
STEPS_PER_DRAW = 12
M32 = 0xFFFFFFFF


def step(s):
    """one xorshift128 step on (x, y, z, w)"""
    x, y, z, w = s
    t = (x ^ (x << 11)) & M32
    return (y, z, w, (w ^ (w >> 19)) ^ (t ^ (t >> 8)))


def draws_from(s, n):
    """n raw draws from state s, and the state after them"""
    out = np.empty(n, dtype=np.uint32)
    x, y, z, w = s
    for i in range(n):
        acc = 0
        for _ in range(STEPS_PER_DRAW):
            t = (x ^ (x << 11)) & M32
            x, y, z = y, z, w
            w = (w ^ (w >> 19)) ^ (t ^ (t >> 8))
            acc += w >> 4
        out[i] = acc
    return out, (x, y, z, w)


def _to_bits(s):
    return np.array([(s[b >> 5] >> (b & 31)) & 1 for b in range(128)], dtype=np.int64)


def _from_bits(v):
    words = [0, 0, 0, 0]
    for b in np.flatnonzero(v):
        words[b >> 5] |= 1 << (int(b) & 31)
    return tuple(words)


@functools.lru_cache(maxsize=None)
def _step_matrix():
    """T with bits(step(s)) = T bits(s) (mod 2): column b is the step of the b-th unit state"""
    T = np.zeros((128, 128), dtype=np.int64)
    for b in range(128):
        e = [0, 0, 0, 0]
        e[b >> 5] = 1 << (b & 31)
        T[:, b] = _to_bits(step(tuple(e)))
    return T


@functools.lru_cache(maxsize=None)
def _step_power(k):
    """T^(2^k) (mod 2)"""
    if k == 0:
        return _step_matrix()
    P = _step_power(k - 1)
    return (P @ P) % 2


def state_at(draw):
    """the generator state after `draw` draws from the seed"""
    e = STEPS_PER_DRAW * int(draw)
    v = _to_bits(SEED)
    k = 0
    while e:
        if e & 1:
            v = (_step_power(k) @ v) % 2
        e >>= 1
        k += 1
    return _from_bits(v)


def window(first, n):
    """raw draws [first, first + n) of the stream"""
    return draws_from(state_at(first), n)[0]


def values(raw):
    """raw sums -> randn() values"""
    return np.asarray(raw, dtype=np.uint32).astype(np.float64) / 268435456.0 - 6.0
