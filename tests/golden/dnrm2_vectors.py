"""Deterministic test vectors for the norm pinning (shared by make_dnrm2_golden.py and tests/test_oracle_norm.py).
A counter-based generator in pure integer arithmetic, so a (seed, n, kind, scale) tuple names the same vector on any
numpy version."""
import numpy as np

_M64 = np.uint64(0xFFFFFFFFFFFFFFFF)


def _splitmix64(z: np.ndarray) -> np.ndarray:
    with np.errstate(over="ignore"):
        z = (z + np.uint64(0x9E3779B97F4A7C15)) & _M64
        z = ((z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)) & _M64
        z = ((z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)) & _M64
        return z ^ (z >> np.uint64(31))


def uniform01(seed: int, n: int) -> np.ndarray:
    with np.errstate(over="ignore"):
        ctr = np.arange(n, dtype=np.uint64) + np.uint64(seed) * np.uint64(0x100000001B3)
    return (_splitmix64(ctr) >> np.uint64(11)).astype(np.float64) * (1.0 / 9007199254740992.0)


def vector(seed: int, n: int, kind: str, scale_exp: int) -> np.ndarray:
    """kind: 'pos' 0.5+u (the bench's x), 'sym' 2u-1, 'masked3' 0.5+u with only every third component kept (what
    x2 = x1 .* (colorvec .== k) looks like for the tridiagonal colouring), 'sparse64' one component in 64 kept, 'const'
    every component 4.79825341824841e-157 (its square is subnormal and rounded by nearly half an ulp, while a sum of
    10^5 of them is a normal number)."""
    u = uniform01(seed, n)
    if kind == "pos":
        x = 0.5 + u
    elif kind == "sym":
        x = 2.0 * u - 1.0
    elif kind == "masked3":
        x = np.where(np.arange(n) % 3 == seed % 3, 0.5 + u, 0.0)
    elif kind == "sparse64":
        x = np.where(np.arange(n) % 64 == seed % 64, 0.5 + u, 0.0)
    elif kind == "const":
        x = np.full(n, 4.79825341824841e-157)
    else:
        raise ValueError(kind)
    return x * (10.0 ** scale_exp)


CASES = (
    [(s, n, k, 0) for s, n in enumerate([32, 33, 39, 40, 47, 64, 100, 255, 1000, 4097, 65536, 100003]) for k in ("pos", "sym", "masked3")]
    + [(100 + s, n, k, e) for s, (n, e) in enumerate([(64, 200), (64, -200), (1000, 150), (1000, -150), (777, 8), (777, -8)])
       for k in ("pos", "sym")]
    + [(200 + s, n, k, 0) for s, n in enumerate([1_000_000, 3_333_334, 10_000_000]) for k in ("pos", "masked3", "sparse64")]
    # beyond the fp64 range of a plain sum of squares: overflowing squares (300), an overflowing norm (307), subnormal
    # squares (-160, partly; -310, -320 all), and the constant vector whose subnormal squares sum to a normal number
    + [(300 + s, n, k, e) for s, (n, e) in enumerate([(64, 300), (1000, 307), (1000, -160), (64, -310), (100, -320)])
       for k in ("pos", "sym")]
    + [(310, 100_000, "const", 0)]
)
