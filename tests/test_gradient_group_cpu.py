"""Host side of the multi-GPU gradient (no GPU): the column partition of a dense group against a restatement of its rule,
the argument checks GroupGradient makes before it touches a device, and the Julia binding's group_gradient methods."""
import re
from pathlib import Path

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent
JL = ROOT / "finitediff.jl_b200" / "julia" / "FiniteDiffB200.jl"


@pytest.fixture(scope="module")
def fdist():
    import _bootstrap
    _bootstrap.load_package()
    from finitediff_jl_b200 import distributed
    return distributed


def restated(n, world):
    """member r owns the columns j with j // ceil(n / world) == r (an empty member sits at n)"""
    p = -(-n // world)
    owner = np.arange(n) // max(p, 1)
    out = []
    for r in range(world):
        cols = np.flatnonzero(owner == r)
        out.append((int(cols[0]), int(cols[-1]) + 1) if cols.size else (n, n))
    return out


def test_partition_matches_the_rule(fdist):
    pairs = [(n, w) for n in list(range(0, 70)) + [1021, 1024, 1029, 20000, 100000] for w in range(1, 10)]
    pairs += [(n, 64) for n in (0, 1, 63, 64, 65, 4095)]
    for n, world in pairs:
        got = fdist.dense_column_blocks(n, world)
        assert got == restated(n, world), (n, world)
        assert got[0][0] == 0 and got[-1][1] == n
        assert all(a[1] == b[0] for a, b in zip(got, got[1:])), (n, world)          # contiguous, in member order
        sizes = [e - b for b, e in got]
        assert sum(sizes) == n and max(sizes) == -(-n // world), (n, world)         # no member above ceil(n / world)
        empty = [r for r, s in enumerate(sizes) if s == 0]
        assert empty == list(range(world - len(empty), world)), (n, world)          # only trailing members are empty
        if n < world:
            assert sizes == [1] * n + [0] * (world - n), (n, world)


def test_partition_refuses_bad_sizes(fdist):
    with pytest.raises(ValueError):
        fdist.dense_column_blocks(-1, 2)
    with pytest.raises(ValueError):
        fdist.dense_column_blocks(4, 0)


def test_constructor_validation_needs_no_device(fdist):
    for n in (-1, 1.5, "3", None, True):
        with pytest.raises(ValueError):
            fdist.GroupGradient(n, [0, 0])
    with pytest.raises(ValueError):
        fdist.GroupGradient(4, [])
    for fdtype in ("hcentral", "backward", 7):
        with pytest.raises(ValueError):
            fdist.GroupGradient(4, [0, 0], fdtype)


def test_run_validation_needs_no_device(fdist):
    g = object.__new__(fdist.GroupGradient)         # the state run() reads before any device work
    g.n, g.devices, g.root = 4, [0, 0], torch.device("cuda", 0)
    f = lambda v: (v * v).sum()
    x = torch.zeros(4, dtype=torch.float64)
    with pytest.raises(ValueError):
        g.run([f], x, x)                              # one f per member
    with pytest.raises(TypeError):
        g.run([f, f], x, x)                           # host tensors: the group has no CPU path
    with pytest.raises(TypeError):
        g.run([f, f], x.float(), x)


def _jl_body(name):
    src = JL.read_text()
    m = re.search(r"\nfunction " + re.escape(name) + r"\(.*?\n(.*?)\nend\n", src, flags=re.S)
    assert m, name
    return m.group(0)


def test_julia_binding_has_group_gradient():
    create = _jl_body("group_gradient")
    assert "fdb_group_create_dense" in create
    # m = 1, n, ldJ = 1: the gradient is the dense group with df as a 1 x n J
    assert re.search(r"pointer\(devices\),\s*1,\s*n,\s*1,\s*opts\)", create)
    run = _jl_body("group_gradient!")
    assert "fdb_group_jacobian" in run
    # forward mode: f(x) once, by fs[1] at the root, unless fx is given; the members get it as f_in
    assert "scalar_f(fs[1])(f_in, x)" in run and "FDB_FORWARD" in run
    assert "pointer(f_in)" in run
