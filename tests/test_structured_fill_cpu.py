"""Host side of tests/test_gpu_structured_fill.py (no GPU): its ELL f has exactly the mirror's entry set for every
structure and target there, its storage decoders put each (row, column) in the mirror's slot, and the CPU oracle
driven by that f lands within the analytic tolerance in forward, central and complex-step mode, so that the GPU
file's value check is neither vacuous nor too tight.  A misaddressed slot fails the check."""
import numpy as np
import pytest

from test_block_dense_plan_cpu import _hook_entries
from test_gpu_structured_fill import (BB_STRUCTS, BD_MANY, BD_PAST, BD_STAGING, BD_STRUCTS, DENSE, DG_SIZES, EDGE_TARGETS,
                                      FD, PACKED, Ell, bd_tile_spans, block_band_entries, block_dense_entries,
                                      check_values, colorings, diagonal_entries, dg_closed, greedy_coloring, host_x,
                                      relabel, tridiag_colour_sum)


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


# ------------------------------------------------------------------------------------------------ block-dense storage
def _all_bd():
    out = list(BD_STRUCTS) + list(BD_MANY)
    out += [(f"edge{i}", s) for i, (k, s) in enumerate(EDGE_TARGETS) if k == "block_dense"]
    out += [("colour_tables", ([3, 0, 4, 2], 1, 1))]
    out += [(name, (rb, 0, 0)) for name, rb, _ in BD_STAGING]
    return out


@pytest.mark.parametrize("name,s", _all_bd(), ids=[c[0] for c in _all_bd()])
def test_block_dense_decoder_and_ell_are_the_mirror_entry_set(pkg, name, s):
    rb, l, u = s
    B = pkg.BlockSkylineMatrix(rb, rb, (l, u), device="cpu")
    rows, cols, slots, length = block_dense_entries(rb, l, u)
    assert length == B.j_len
    assert np.array_equal(np.sort(slots), np.arange(length)), name        # every slot is one structural entry
    mr, mc, ms = B.findstructralnz()
    hr, hc, hs, hlen = _hook_entries(rb, l, u) if length < 200_000 else (mr, mc, ms, length)
    assert hlen == length
    a = _sorted(rows + 1, cols + 1, slots + 1)
    for x, y, z in zip(a, _sorted(mr, mc, ms), _sorted(hr, hc, hs)):
        assert np.array_equal(x, y) and np.array_equal(x, z), name
    ell = Ell(B.n, rows, cols, 1)
    nz = ell.coef != 0
    key = np.sort((np.broadcast_to(np.arange(B.n), ell.cols.shape)[nz] * B.n + ell.cols[nz]).astype(np.int64))
    assert np.array_equal(key, np.sort(rows * B.n + cols)), name


def test_block_dense_staging_spans():
    """The tiles of the staging-boundary structures span 255, 256 and 257 block columns, every one of them (the last,
    partial tile at most that many), so the staged and unstaged searches meet at kBdStage = 256."""
    for name, rb, span in BD_STAGING:
        spans = bd_tile_spans(rb, 0, 0)
        assert len(spans) > 2 and set(spans[:-1].tolist()) == {span} and spans[-1] <= span, (name, spans)
    # blocks of one slot, hundreds per tile: far past the boundary
    assert bd_tile_spans([1] * 3000, 0, 0)[0] == 1024
    # the replica agrees with a slot-by-slot walk on a small irregular structure
    rb, l, u = [3, 0, 40, 1, 1, 2, 0, 25, 7], 1, 2
    _, cols, slots, length = block_dense_entries(rb, l, u)
    off = np.concatenate([[0], np.cumsum(rb)])
    bcol = np.searchsorted(off, np.arange(sum(rb)), side="right") - 1
    col_of_slot = np.empty(length, np.int64)
    col_of_slot[slots] = bcol[cols]
    walk = [col_of_slot[min(s + 1023, length - 1)] - col_of_slot[s] + 1 for s in range(0, length, 1024)]
    assert bd_tile_spans(rb, l, u, 1024).tolist() == walk


def test_block_dense_past_2_31_decoding():
    """The int64 decode of the past-2^31 test (slab start, column, row) agrees with the decoder on a small structure
    of the same shapes, and the structures reach the sizes they are named for."""
    for name, rb, l, u in BD_PAST:
        N = len(rb)
        off = np.concatenate([[0], np.cumsum(rb)]).astype(np.int64)
        h = off[np.minimum(np.arange(N) + l, N - 1) + 1] - off[np.maximum(np.arange(N) - u, 0)]
        start = np.concatenate([[0], np.cumsum(h * np.asarray(rb, np.int64))])
        assert start[-1] > 2 ** 31, name
        if name == "one_slab":
            assert 2 ** 31 < start[-1] < 2 ** 32
        else:
            assert (start < 2 ** 31).any() and (start > 2 ** 31).any() and h.max() * max(rb) < 2 ** 31
    rb, l, u = [5, 3, 6, 2], 1, 1
    rows, cols, slots, length = block_dense_entries(rb, l, u)
    N = len(rb)
    off = np.concatenate([[0], np.cumsum(rb)]).astype(np.int64)
    K0 = np.maximum(np.arange(N) - u, 0)
    h = off[np.minimum(np.arange(N) + l, N - 1) + 1] - off[K0]
    start = np.concatenate([[0], np.cumsum(h * np.asarray(rb, np.int64))])
    J = np.searchsorted(start[:N], slots, side="right") - 1
    rel = slots - start[J]
    assert np.array_equal(off[J] + rel // h[J], cols) and np.array_equal(off[K0[J]] + rel % h[J], rows)
    # the closed-form tridiagonal value: -2 on the diagonal, 1 beside it, under the identity colouring
    n = 8
    r = np.arange(n)
    assert np.array_equal(tridiag_colour_sum(r, r, np.arange(1, n + 1), n), np.full(n, -2.0))


CPU_BD = ["empty_inner", "empty_but_one", "l_ne_u", "wide_bands", "size1", "uniform6"]


@pytest.mark.parametrize("name", CPU_BD)
@pytest.mark.parametrize("fdtype", ["forward", "central", "complex"])
def test_oracle_within_analytic_tolerance_block_dense(pkg, oracle, name, fdtype):
    s = dict(BD_STRUCTS)[name]
    st = block_dense_entries(*s)
    n = sum(s[0])
    ell = Ell(n, st[0], st[1], 13)
    x = host_x(n, 14)
    closed = pkg.BlockSkylineMatrix(s[0], s[0], (s[1], s[2]), device="cpu").matrix_colors()
    for cvname, (cv, valid) in colorings(closed, n, st[0], st[1], np.random.default_rng(1)).items():
        for kw in ([{}] if fdtype == "complex" else [{}, {"dir": -1.0}, {"relstep": 1e-5, "absstep": 1e-9}]):
            ref, eps = _oracle(oracle, st, n, ell, x, fdtype, cv, kw)
            check_values(ref, st, ell, x, cv, eps, fdtype, valid, f"{name} {fdtype} {cvname} {kw}")


@pytest.mark.parametrize("fdtype", ["forward", "central", "complex"])
def test_block_dense_misaddressed_slot_fails_the_check(pkg, oracle, fdtype):
    """Every block-dense slot is structural: swapping two slots of one column, or moving a value to the next slot of
    its slab, or zeroing one, fails check_values."""
    s = dict(BD_STRUCTS)["l_ne_u"]
    st = block_dense_entries(*s)
    rows, cols, slots, length = st
    n = sum(s[0])
    ell = Ell(n, rows, cols, 13)
    x = host_x(n, 14)
    cv = pkg.BlockSkylineMatrix(s[0], s[0], (s[1], s[2]), device="cpu").matrix_colors()
    ref, eps = _oracle(oracle, st, n, ell, x, fdtype, cv)
    check_values(ref, st, ell, x, cv, eps, fdtype, True, "unchanged")
    same = np.flatnonzero(cols == cols[0])
    i, j = slots[same[0]], slots[same[1]]
    assert ref[i] != ref[j]
    for what, edit in (("swap", lambda J: J.__setitem__([i, j], J[[j, i]])),
                       ("shifted", lambda J: J.__setitem__(slice(i, i + 2), J[[i + 1, i]])),
                       ("zeroed", lambda J: J.__setitem__(i, 0.0))):
        bad = ref.copy()
        edit(bad)
        with pytest.raises(AssertionError):
            check_values(bad, st, ell, x, cv, eps, fdtype, True, what)
