"""The two CPU restatements of the out-of-place forms against each other: the C restatement (oop_oracle/) and the
line-by-line numpy transcription (tests/_literal_oop.py), written independently, on a few hundred random problems over
every result kind, forward / central / complex, dir = +-1 and 0.3, step overrides, f_in given or not, the cached and
cache-less forms, valid and invalid colourings and colour 0.  Both call the same f, so they must see the same points in
the same order and return the same bits.  Half the problems take the step sizes from their own norms, on x whose colour
norms are exact (integers over 2^5), so that the norm's summation order cannot matter; the other half feed both the same
step sizes on general x with signed zeros and NaN."""
import numpy as np
import pytest

import _literal_oop as LO
from oop_oracle import fd_oop_oracle as OO


def bits_equal(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return a.shape == b.shape and bool(np.all((a.view(np.uint64) == b.view(np.uint64)) | (np.isnan(a) & np.isnan(b))))


class Rec:
    def __init__(self, f):
        self.f, self.points = f, []

    def __call__(self, x):
        self.points.append(np.array(x, copy=True))
        return self.f(x)


def _problem(seed):
    rng = np.random.default_rng(seed)
    fd = ["forward", "central", "complex"][seed % 3]
    n = int(rng.integers(1, 10))
    csc = bool(rng.integers(0, 2))
    m = n if csc else int(rng.integers(1, 10))
    p1, p2, p3 = (rng.integers(0, n, m) for _ in range(3))
    a, b = rng.uniform(-2, 2, m), rng.uniform(-2, 2, m)
    f = lambda x: (a * x[p1]) * x[p2] + b * x[p3]
    exact = seed % 2 == 0
    if exact:
        x = rng.integers(-40, 40, n) * 2.0 ** -5
    else:
        x = rng.uniform(-1.5, 1.5, n)
        x[rng.random(n) < 0.2] = -0.0
        if rng.random() < 0.15:
            x[rng.integers(0, n)] = np.nan
    kw = {"dir": [1.0, -1.0, 0.3][int(rng.integers(0, 3))]}
    steps = [(None, None), (1e-3, 0.0), (0.0, 1e-4), (-1e-3, 1e-160), (1.0, None)][int(rng.integers(0, 5))]
    kw["relstep"], kw["absstep"] = steps
    f_in = f(x) if (fd == "forward" and rng.random() < 0.4) else None
    kw["cacheless"] = bool(rng.random() < 0.25)
    if csc:
        A = rng.random((m, n)) < 0.4
        A[np.arange(min(m, n)), np.arange(min(m, n))] = True
        cp = np.concatenate([[0], np.cumsum(A.sum(axis=0))]).astype(np.int64) + 1
        rv = np.concatenate([np.flatnonzero(A[:, c]) for c in range(n)]).astype(np.int64) + 1
        kw["sparsity"] = (m, n, cp, rv)
        kw["colorvec"] = rng.integers(0 if rng.random() < 0.2 else 1, 4, n)
        if kw["colorvec"].max() < 1:
            kw["colorvec"][0] = 1
        if rng.random() < 0.5:
            kw["jac_prototype"] = ("sparse", m, n)
        if fd != "complex" and not exact:
            kw["eps_override"] = list(rng.uniform(-1e-2, 1e-2, int(kw["colorvec"].max())))
    else:
        C = int(rng.integers(1, n + 1))
        if rng.random() < 0.5:
            kw["colorvec"] = np.concatenate([[C], rng.integers(1, C + 1, n - 1)])
        else:
            kw["colorvec"] = np.arange(1, n + 1)
            C = n
        r = rng.random()
        if r < 0.33:
            kw["jac_prototype"] = ("dense", m, C + int(rng.integers(0, 3)))
        elif r < 0.66:
            kw["jac_prototype"] = ("sparse", m, C + int(rng.integers(0, 3)))
    return fd, f, x, f_in, kw


@pytest.mark.parametrize("seed", range(300))
def test_c_restatement_matches_the_transcription(seed):
    fd, f, x, f_in, kw = _problem(seed)
    rl, ro = Rec(f), Rec(f)
    outs = []
    for impl, rec, extra in ((LO, rl, {}), (OO, ro, {"m": np.asarray(f(x)).size})):
        try:
            outs.append(impl.jacobian_oop(rec, x.copy(), fd, f_in, **kw, **extra))
        except (LO.MakeJiError, OO.OracleThrows):
            outs.append("throws")
    assert (outs[0] == "throws") == (outs[1] == "throws"), (seed, outs)
    if outs[0] != "throws":
        assert outs[0][0] == outs[1][0]
        if outs[0][0] == "dense":
            assert bits_equal(outs[0][1], outs[1][1]), seed
        else:
            assert outs[0][1:3] == outs[1][1:3]
            assert np.array_equal(outs[0][3], outs[1][3]) and np.array_equal(outs[0][4], outs[1][4]), seed
            assert bits_equal(outs[0][5], outs[1][5]), seed
    assert len(rl.points) == len(ro.points), seed
    for p, q in zip(rl.points, ro.points):
        if np.iscomplexobj(p) or np.iscomplexobj(q):
            assert bits_equal(np.real(p), np.real(q)) and bits_equal(np.imag(p), np.imag(q)), seed
        else:
            assert bits_equal(p, q), seed


@pytest.mark.parametrize("cacheless", [False, True])
@pytest.mark.parametrize("fd", ["forward", "central", "complex"])
@pytest.mark.parametrize("proto", ["raw", "dense", "sparse"])
@pytest.mark.parametrize("colour", [0, -2])
def test_dense_branch_without_colours(colour, proto, fd, cacheless):
    """sparsity = nothing with maximum(colorvec) < 1: the colour loop is empty, so both restatements return
    zero(jac_prototype) (+0.0 everywhere, or colptr all 1 and nnz 0) after f(x) in forward mode; without a prototype the
    result is sized by mapreduce over the empty range, which throws"""
    rng = np.random.default_rng(7)
    m, n = 4, 3
    p1 = rng.integers(0, n, m)
    f = lambda x: x[p1] * x[p1]
    x = np.array([0.5, -0.0, 1.25])
    kw = {"colorvec": np.full(n, colour, np.int64), "cacheless": cacheless}
    if proto != "raw":
        kw["jac_prototype"] = (proto, m, n + 1)
    rl, ro = Rec(f), Rec(f)
    outs = []
    for impl, rec, extra in ((LO, rl, {}), (OO, ro, {"m": m})):
        try:
            outs.append(impl.jacobian_oop(rec, x.copy(), fd, None, **kw, **extra))
        except (LO.MakeJiError, ValueError):
            outs.append("throws")
    if proto == "raw":
        assert outs == ["throws", "throws"]
        return
    calls = 1 if (fd == "forward" or cacheless) else 0          # :299-300, or the cache-less form's own f(x) (:250-251)
    assert len(rl.points) == len(ro.points) == calls
    for out in outs:
        if proto == "dense":
            assert out[0] == "dense" and bits_equal(out[1], np.zeros((m, n + 1)))
        else:
            assert out[0] == "sparse" and out[1:3] == (m, n + 1)
            assert np.array_equal(out[3], np.ones(n + 2, np.int64)) and out[4].size == 0 and out[5].size == 0


@pytest.mark.parametrize("seed", range(60))
def test_c_jvp_matches_the_transcription(seed):
    rng = np.random.default_rng(1000 + seed)
    fd = ["forward", "central"][seed % 2]
    n, m = int(rng.integers(0, 9)), int(rng.integers(0, 9))
    p1 = rng.integers(0, max(n, 1), m)
    f = (lambda x: x[p1] * x[p1] + 0.5 * x[p1]) if n else (lambda x: np.zeros(m))
    x = rng.integers(-40, 40, n) * 2.0 ** -5                      # x.v exact in any order
    v = rng.integers(-8, 8, n) * 2.0 ** -3
    kw = {"dir": [1.0, -1.0, 0.3][seed % 3], "cacheless": seed % 4 == 1}
    kw["relstep"], kw["absstep"] = [(None, None), (1e-3, 0.0), (0.0, 1e-4)][seed % 3]
    f_in = f(x) if (fd == "forward" and seed % 5 == 0) else None
    rl, ro = Rec(f), Rec(f)
    a, ea = LO.jvp_oop(rl, x, v, fd, f_in, **kw)
    b, eb = OO.jvp_oop(ro, x, v, fd, f_in, m=m, **kw)
    assert bits_equal([ea], [eb]) and bits_equal(a, b), seed
    assert len(rl.points) == len(ro.points) and all(bits_equal(p, q) for p, q in zip(rl.points, ro.points))
