"""prng.py -- the reference's random stream on the host: Threefry-2x32 counter PRNG, key splitting and N(0,1) draws.

The reference hands `rng_key` to `jax.random.split` (one key per hyper-parameter draw, gpax/models/gp.py:391) and each
key to `numpyro.distributions.MultivariateNormal.sample`, which draws `jax.random.normal(key, (n, P))` and returns
`mean + chol(cov) eps` (gp.py:292).  Reproducing y_sampled for a given key therefore needs JAX's bit stream, not any
N(0,1) generator.  This module restates the published algorithm (Salmon et al., "Parallel random numbers: as easy as
1, 2, 3", SC'11, Threefry-2x32 with 20 rounds, and the way JAX's `jax/_src/prng.py` / `random.py` turn its output into
keys, uniforms and normals) in NumPy.  JAX is not installed in this image, so the restatement is pinned to the known
answers JAX itself publishes (tests/test_prng.py): the Random123 known-answer vector that JAX's own test-suite uses,
`split(PRNGKey(0))` and `normal(PRNGKey(0), (1,))` from the JAX PRNG documentation.

Two details follow the JAX version the reference was written against (0.4.x): keys are split and bits are drawn with
the original ("non-partitionable") counter layout.  `partitionable=True` gives the layout JAX >= 0.5 uses by default.
The inverse error function is SciPy's (float64, then rounded): XLA's float32 polynomial differs from it by at most a
few ulp, i.e. draws agree with the reference's to ~1e-6 relative in float32 and exactly in the bit stream.
"""
from __future__ import annotations

import numpy as np
from scipy.special import erfinv

_U32 = np.uint32
_ROT = ((13, 15, 26, 6), (17, 29, 16, 24))


def _rotl(x, r):
    return (x << _U32(r)) | (x >> _U32(32 - r))


def threefry2x32(k1, k2, x0, x1):
    """Threefry-2x32, 20 rounds, on arrays of counters (x0, x1) under the key (k1, k2); returns two uint32 arrays."""
    with np.errstate(over="ignore"):
        k1, k2 = _U32(k1), _U32(k2)
        ks = (k1, k2, _U32(k1 ^ k2 ^ _U32(0x1BD11BDA)))
        x0 = np.asarray(x0, dtype=_U32) + ks[0]
        x1 = np.asarray(x1, dtype=_U32) + ks[1]
        for i in range(5):
            for r in _ROT[i % 2]:
                x0 = x0 + x1
                x1 = _rotl(x1, r) ^ x0
            x0 = x0 + ks[(i + 1) % 3]
            x1 = x1 + ks[(i + 2) % 3] + _U32(i + 1)
    return x0, x1


def _threefry_2x32(key, count):
    """jax/_src/prng.py threefry_2x32: the counter array is cut in two halves that form the two Threefry words."""
    count = np.asarray(count, dtype=_U32)
    flat = count.ravel()
    odd = flat.size % 2
    if odd:
        flat = np.concatenate([flat, np.zeros(1, _U32)])
    h = flat.size // 2
    a, b = threefry2x32(key[0], key[1], flat[:h], flat[h:])
    out = np.concatenate([a, b])
    return (out[:-1] if odd else out).reshape(count.shape)


def _iota_2x32(shape):
    idx = np.arange(int(np.prod(shape, dtype=np.int64)), dtype=np.uint64).reshape(shape)
    return (idx >> np.uint64(32)).astype(_U32), (idx & np.uint64(0xFFFFFFFF)).astype(_U32)


def as_key(rng_key) -> np.ndarray:
    """uint32[2] key from an int seed (as jax.random.PRNGKey), a uint32 pair, or a jax key array."""
    if isinstance(rng_key, (int, np.integer)):
        return PRNGKey(int(rng_key))
    arr = np.asarray(rng_key)
    if arr.dtype.kind not in "iu" or arr.size != 2:
        raise TypeError("rng_key must be an int seed or a pair of 32-bit integers (a jax.random.PRNGKey)")
    return (arr.reshape(2).astype(np.int64) & 0xFFFFFFFF).astype(_U32)


def PRNGKey(seed: int) -> np.ndarray:
    """jax.random.PRNGKey: the 64-bit seed as (high word, low word)."""
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    return np.array([seed >> 32, seed & 0xFFFFFFFF], dtype=_U32)


def split(key, num: int = 2, partitionable: bool = False) -> np.ndarray:
    """jax.random.split: `num` new keys, shape (num, 2)."""
    key = as_key(key)
    if partitionable:
        hi, lo = _iota_2x32((num,))
        a, b = threefry2x32(key[0], key[1], hi, lo)
        return np.stack([a, b], axis=1)
    return _threefry_2x32(key, np.arange(2 * num, dtype=_U32)).reshape(num, 2)


def random_bits(key, bit_width: int, shape, partitionable: bool = False) -> np.ndarray:
    """jax.random.bits for 32- and 64-bit words."""
    key = as_key(key)
    shape = tuple(int(s) for s in shape)
    size = int(np.prod(shape, dtype=np.int64))
    if bit_width not in (32, 64):
        raise ValueError("bit_width must be 32 or 64")
    if partitionable:
        hi, lo = _iota_2x32(shape)
        a, b = threefry2x32(key[0], key[1], hi, lo)
        if bit_width == 32:
            return a ^ b
        return (a.astype(np.uint64) << np.uint64(32)) | b.astype(np.uint64)
    words = size * bit_width // 32
    bits = _threefry_2x32(key, np.arange(words, dtype=_U32))
    if bit_width == 64:
        bits = (bits[:size].astype(np.uint64) << np.uint64(32)) | bits[size:].astype(np.uint64)
    return bits.reshape(shape)


def uniform(key, shape, dtype=np.float32, minval=0.0, maxval=1.0, partitionable: bool = False) -> np.ndarray:
    """jax.random.uniform: mantissa bits under the exponent of 1.0, minus 1, scaled and clamped from below."""
    dtype = np.dtype(dtype)
    nbits, nmant = (32, 23) if dtype == np.float32 else (64, 52)
    utype = np.uint32 if nbits == 32 else np.uint64
    bits = random_bits(key, nbits, shape, partitionable).astype(utype)
    one = np.array(1.0, dtype).view(utype)
    floats = ((bits >> utype(nbits - nmant)) | one).view(dtype) - dtype.type(1.0)
    lo, hi = dtype.type(minval), dtype.type(maxval)
    return np.maximum(lo, floats * (hi - lo) + lo).astype(dtype)


def randint(key, shape, minval, maxval, partitionable: bool = False) -> np.ndarray:
    """jax.random.randint for int32 results (the JAX 0.4 algorithm): split the key, draw two 32-bit words hi and lo, and
    reduce ((hi % span) * ((2**16 % span)**2 % span) + lo % span) % span in uint32 arithmetic, plus minval; span = 1
    when maxval <= minval (every draw is minval).  JAX is not installed here, so unlike split / normal this restatement
    is not pinned to a value JAX published; it follows the algorithm, not a known answer."""
    shape = tuple(int(s) for s in shape)
    minval, maxval = int(minval), int(maxval)
    k1, k2 = split(key, 2, partitionable)
    hi = random_bits(k1, 32, shape, partitionable)
    lo = random_bits(k2, 32, shape, partitionable)
    span = _U32(maxval - minval if maxval > minval else 1)
    with np.errstate(over="ignore"):
        mult = _U32(2 ** 16) % span
        mult = (mult * mult) % span
        off = ((hi % span) * mult + lo % span) % span
    return (off.astype(np.int64) + minval).astype(np.int32)


def normal(key, shape, dtype=np.float32, partitionable: bool = False) -> np.ndarray:
    """jax.random.normal: sqrt(2) * erfinv(u), u uniform on (-1, 1)."""
    dtype = np.dtype(dtype)
    lo = np.nextafter(dtype.type(-1.0), dtype.type(0.0))
    u = uniform(key, shape, dtype, lo, 1.0, partitionable)
    return (dtype.type(np.sqrt(2.0)) * erfinv(u.astype(np.float64)).astype(dtype)).astype(dtype)


def mvn_eps(rng_key, num_draws: int, n: int, P: int, dtype=np.float32, partitionable: bool = False) -> np.ndarray:
    """The standard normals behind the reference's y_sampled: keys = split(rng_key, num_draws) (gp.py:391), then
    normal(keys[s], (n, P)) per draw (numpyro MultivariateNormal.sample, called at gp.py:292).  Shape (S, n, P), float64."""
    keys = split(rng_key, num_draws, partitionable)
    out = np.empty((num_draws, n, P))
    for s in range(num_draws):
        out[s] = normal(keys[s], (n, P), dtype, partitionable)
    return out
