"""Host side of tests/test_gpu_structured_fill.py (no GPU): its ELL f has exactly the mirror's entry set for every
structure and target there, its storage decoders put each (row, column) in the mirror's slot, and the CPU oracle
driven by that f lands within the analytic tolerance in forward, central and complex-step mode, so that the GPU
file's value check is neither vacuous nor too tight.  A misaddressed slot fails the check."""
import numpy as np
import pytest

from test_gpu_structured_fill import (BB_STRUCTS, DENSE, DG_SIZES, EDGE_TARGETS, FD, PACKED, Ell, block_band_entries,
                                      check_values, colorings, diagonal_entries, dg_closed, greedy_coloring, host_x,
                                      relabel)


@pytest.fixture(scope="module")
def pkg():
    import _bootstrap
    return _bootstrap.load_package()


def _all_bb():
    out = list(BB_STRUCTS)
    out += [(f"edge{i}", s) for i, (k, s) in enumerate(EDGE_TARGETS) if k == "bb"]
    out += [("many_colours", ([41] * 25, 12, 12, 20, 20, False)), ("colour_tables", ([3, 0, 4, 2], 1, 1, 1, 1, False))]
    return out


def _mirror_bb(pkg, s):
    rb, l, u, lam, mu, dense = s
    if dense:
        return pkg.BlockBandedMatrix(rb, rb, (l, u), device="cpu")
    return pkg.BandedBlockBandedMatrix(rb, rb, (l, u), (lam, mu), device="cpu")


def _sorted(rows, cols, slots):
    o = np.argsort(slots, kind="stable")
    return rows[o], cols[o], slots[o]


@pytest.mark.parametrize("name,s", _all_bb(), ids=[c[0] for c in _all_bb()])
def test_block_band_decoder_and_ell_are_the_mirror_entry_set(pkg, name, s):
    B = _mirror_bb(pkg, s)
    rows, cols, slots, length = block_band_entries(*s)
    assert length == B.w * B.n == B.data.numel()
    mr, mc, ms = B.findstructralnz()
    a, b = _sorted(rows + 1, cols + 1, slots + 1), _sorted(mr, mc, ms)
    for x, y in zip(a, b):
        assert np.array_equal(x, y), name
    ell = Ell(B.n, rows, cols, 1)
    pattern = {(int(r), int(c)) for p in range(ell.K) for r, c in zip(range(B.n), ell.cols[p])}
    assert pattern == set(zip((mr - 1).tolist(), (mc - 1).tolist())), name
    # padding repeats the row's slot-0 column with coefficient +0.0; every listed (row, column) has its own coefficient
    for r in range(B.n):
        seen = [int(c) for c, a in zip(ell.cols[:, r], ell.coef[:, r]) if a != 0.0]
        assert len(seen) == len(set(seen))
        pad = ell.coef[:, r] == 0.0
        assert np.all(ell.coef[:, r][pad].view(np.uint64) == 0) and np.all(ell.cols[:, r][pad] == ell.cols[0, r])
    assert np.all(np.abs(ell.coef[ell.coef != 0]) >= 0.5) and np.all(np.abs(ell.coef) <= 2.0)


def _mirror_dg(pkg, kind, n):
    base = kind[len("dense_"):] if kind.startswith("dense_") else kind
    return {"diag": lambda: pkg.Diagonal(n, device="cpu"), "bidiag_U": lambda: pkg.Bidiagonal(n, "U", device="cpu"),
            "bidiag_L": lambda: pkg.Bidiagonal(n, "L", device="cpu"), "symtri": lambda: pkg.SymTridiagonal(n),
            "tri": lambda: pkg.Tridiagonal(n, device="cpu")}[base]()


@pytest.mark.parametrize("kind", PACKED + DENSE)
def test_diagonal_decoder_and_ell_are_the_mirror_entry_set(pkg, kind):
    for n in sorted(set(DG_SIZES + [130, 301, 600, 700, 61])):
        rows, cols, slots, length = diagonal_entries(kind, n)
        M = _mirror_dg(pkg, kind, n)
        mr, mc, ms = M.findstructralnz()
        if kind in PACKED:
            assert length == M.buf.numel()
            a, b = _sorted(rows + 1, cols + 1, slots + 1), _sorted(mr, mc, ms)
            for x, y in zip(a, b):
                assert np.array_equal(x, y), (kind, n)
        else:
            assert set(zip(rows.tolist(), cols.tolist())) == set(zip((mr - 1).tolist(), (mc - 1).tolist()))
            assert np.array_equal(slots, cols * n + rows) and length == n * n
        ell = Ell(n, rows, cols, 2)
        pattern = {(r, int(c)) for p in range(ell.K) for r, c in enumerate(ell.cols[p])}
        assert pattern == set(zip(rows.tolist(), cols.tolist())), (kind, n)


def test_colourings_are_valid_and_relabelled(pkg):
    """matrix_colors and the greedy colouring are distance-2 valid on each structure (the analytic check relies on it),
    and the relabelled colouring keeps each colour's column set under another label."""
    cases = [(name, block_band_entries(*s), _mirror_bb(pkg, s).matrix_colors()) for name, s in _all_bb()]
    cases += [(f"{k} n={n}", diagonal_entries(k, n), dg_closed(k, n)) for k in PACKED for n in (1, 2, 3, 700)]
    for name, (rows, cols, _, _), closed in cases:
        n = len(closed)
        for cv in (closed, greedy_coloring(n, rows, cols, np.random.default_rng(0))):
            key = rows * (int(cv.max()) + 1) + cv[cols]
            assert len(np.unique(key)) == len(key), f"{name}: two columns of one colour share a row"
        rl = relabel(closed)
        assert len({(a, b) for a, b in zip(closed.tolist(), rl.tolist())}) == len(set(closed.tolist())), name
        if closed.max() > 1:
            assert not np.array_equal(rl, closed), name


def _oracle(oracle, st, n, ell, x, fdtype, cv, kw=None):
    rows, cols, slots, length = st
    P = oracle.Problem.coo_to_slots(n, n, rows + 1, cols + 1, slots + 1, length)
    ref = np.full(length, np.nan)
    kw = kw or {}
    if fdtype == "complex":
        oracle.jacobian_complex(P, ref, oracle.native_fn("synth_ellrows_c"), x.copy(), colorvec=cv, ctx=ell.octx(oracle))
        return ref, None
    r = oracle.jacobian(P, ref, oracle.native_fn("synth_ellrows"), x.copy(), fdtype=FD[fdtype], colorvec=cv,
                        ctx=ell.octx(oracle), **kw)
    return ref, r["eps"]


CPU_BB = ["empty_inner", "empty_but_one", "l_ne_u_wide", "w9_big_blocks", "one_block_wide", "dense_blocks",
          "size1_nonuniform"]


@pytest.mark.parametrize("name", CPU_BB)
@pytest.mark.parametrize("fdtype", ["forward", "central", "complex"])
def test_oracle_within_analytic_tolerance_block_band(pkg, oracle, name, fdtype):
    s = dict(BB_STRUCTS)[name]
    st = block_band_entries(*s)
    n = sum(s[0])
    ell = Ell(n, st[0], st[1], 11)
    x = host_x(n, 12)
    closed = _mirror_bb(pkg, s).matrix_colors()
    for cvname, (cv, valid) in colorings(closed, n, st[0], st[1], np.random.default_rng(1)).items():
        for kw in ([{}] if fdtype == "complex" else [{}, {"dir": -1.0}, {"relstep": 1e-5, "absstep": 1e-9}]):
            ref, eps = _oracle(oracle, st, n, ell, x, fdtype, cv, kw)
            check_values(ref, st, ell, x, cv, eps, fdtype, valid, f"{name} {fdtype} {cvname} {kw}")


@pytest.mark.parametrize("kind", PACKED)
@pytest.mark.parametrize("fdtype", ["forward", "central", "complex"])
def test_oracle_within_analytic_tolerance_diagonals(oracle, kind, fdtype):
    for n in (1, 2, 3, 700):
        st = diagonal_entries(kind, n)
        ell = Ell(n, st[0], st[1], n)
        x = host_x(n, n + 1)
        for cvname, (cv, valid) in colorings(dg_closed(kind, n), n, st[0], st[1], np.random.default_rng(n)).items():
            ref, eps = _oracle(oracle, st, n, ell, x, fdtype, cv)
            check_values(ref, st, ell, x, cv, eps, fdtype, valid, f"{kind} {fdtype} n={n} {cvname}")


@pytest.mark.parametrize("fdtype", ["forward", "central", "complex"])
def test_misaddressed_slot_fails_the_check(pkg, oracle, fdtype):
    """Swapping the values of two structural slots, moving one to a slot outside the structure, or zeroing one slot
    each fail check_values: the tolerance is far below the spread of the coefficients."""
    s = dict(BB_STRUCTS)["empty_inner"]
    st = block_band_entries(*s)
    rows, cols, slots, length = st
    n = sum(s[0])
    ell = Ell(n, rows, cols, 11)
    x = host_x(n, 12)
    cv = _mirror_bb(pkg, s).matrix_colors()
    ref, eps = _oracle(oracle, st, n, ell, x, fdtype, cv)
    check_values(ref, st, ell, x, cv, eps, fdtype, True, "unchanged")
    # two slots of one column, holding different values
    c0 = cols[0]
    same = np.flatnonzero(cols == c0)
    i, j = same[0], same[1]
    assert ref[slots[i]] != ref[slots[j]]
    inside = np.zeros(length, bool)
    inside[slots] = True
    outside = int(np.flatnonzero(~inside)[0])
    for what, edit in (("swap", lambda J: J.__setitem__([slots[i], slots[j]], J[[slots[j], slots[i]]])),
                       ("moved out", lambda J: J.__setitem__([outside, slots[i]], [J[slots[i]], 0.0])),
                       ("-0.0 outside", lambda J: J.__setitem__(outside, -0.0)),
                       ("zeroed", lambda J: J.__setitem__(slots[i], 0.0))):
        bad = ref.copy()
        edit(bad)
        with pytest.raises(AssertionError):
            check_values(bad, st, ell, x, cv, eps, fdtype, True, what)
