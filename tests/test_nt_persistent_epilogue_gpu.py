"""Every epilogue functor of the wgmma NT tiles where each CTA walks many 64-row tiles: the benchmark's 65 536 rows (and
65 573, a ragged last row tile) at the natural persistent grid, and 4 133 rows with the grid capped at 1, 2, 3 and 5
CTAs per column tile (avc_tc_nt_set_max_ctas), so that one CTA walks up to all 65 row tiles, 33 on consumer warpgroup 0
and 32 on warpgroup 1.  That is where the second warpgroup, the turn hand-off, the operand ring's counter and parity
across tiles, the staged loaders, the epilogue ring's chunk counter and the draining of its TMA stores run; the
functor files (test_nt_epilogue_gpu.py, test_nt_store_gpu.py, test_nt_staged_store_gpu.py) run one tile per CTA.
Each run is checked against those files' fp64 formulas and bars, with their sentinels, padding checks and store paths,
and the grid of the launch (avc_tc_nt_last_grid) against the rule restated here.  A row's arithmetic does not depend on
the CTA, warpgroup or tile that computes it, so every output is also bitwise equal across the placements, repeat runs
and the leading rows of the long launches; the short launches use views of the long launch's buffers, so a tensor map
cached for the long launch would write the short one's sentinel rows."""
import ctypes as C
import math

import pytest
import torch

from test_nt_staged_store_gpu import (BAR, CHAIN_SHAPES, EXTRA, SHAPES, _chain_bwd_ref, _chain_ref, _check_f32,
                                      _check_split, _dgrad_ref, _err)
from test_nt_store_gpu import (BAR_D1, BAR_NP1, RELU_SHAPES, STORE_SHAPES, VALUE_SHAPES, _aligned, _check_store,
                               _color0_ref, _relu_mask_ref, _sentinel_split, _split_acc, _value_ref, r4, r8)

M_BENCH = 65536          # the benchmark's rows per NT GEMM: 512 rays x 128 samples
M_BIG = 65573            # ... and a ragged last row tile (37 rows)
M_SMALL = 4133           # 64 whole row tiles and a ragged one
SMS = (132, 114)         # the H100 SXM and PCIe parts
# (M, cap in CTAs per column tile (0: none), the fewest row tiles each warpgroup of a CTA runs (None: see _claim))
PLACEMENTS = [(M_BENCH, 0, None), (M_BIG, 0, None), (M_SMALL, 1, (33, 32)), (M_SMALL, 2, (16, 16)),
              (M_SMALL, 3, (11, 10)), (M_SMALL, 5, (7, 6)), (M_SMALL, 0, (1, 0)), (M_SMALL, 0, (1, 0))]


# ------------------------------------------------------------------------------------------------ the grid rule
def _tiles_n(N):
    bn = 64 if N <= 64 else 128
    return (N + bn - 1) // bn


def _grid(M, N, sms, cap=0):
    """gridDim.x of an NT launch (launch_gemm_tc_nt_kern): at most one CTA per tile and per SM, a whole number per column
    tile; the test cap (CTAs) rounded down to whole CTAs per column tile, at least one."""
    tn = _tiles_n(N)
    g = min((M + 63) // 64 * tn, sms) // tn * tn
    return min(g, max(cap // tn, 1) * tn) if cap > 0 else g


def _walk(M, N, g):
    """(fewest row tiles of warpgroup 0 and 1 on a CTA, most, the warpgroup of the ragged last row tile or None):
    a CTA walks the row tiles m_first, m_first + stride, ..; its j-th tile goes to warpgroup j & 1."""
    tm, stride = (M + 63) // 64, g // _tiles_n(N)
    n = [len(range(r, tm, stride)) for r in range(stride)]
    lo = (min((k + 1) // 2 for k in n), min(k // 2 for k in n))
    hi = (max((k + 1) // 2 for k in n), max(k // 2 for k in n))
    return lo, hi, ((tm - 1) // stride) & 1 if M % 64 else None


def _claim(M, N, cap, claim):
    # at the natural grid of 132 SMs: 15-16 row tiles per CTA with two column tiles, 7-8 with one
    return claim if claim is not None else (8, 7) if _tiles_n(N) == 2 else (4, 3)


# ------------------------------------------------------------------------------------------------ the cases
class Case:
    """One (kind, shape): kind as avc_tc_epi_test takes it ('plain': avc_tc_gemm_nt_test), N, K, the widths, the store
    path the shape takes, whether the fp64 accumulator is the exact product (the backward files) or the product of the
    split operands (the store file), and make(g) -> (launch arguments, check(M, acc) -> {name: error})."""

    def __init__(self, name, kind, N, K, ring, make, ldx=8, ld2=8, Nv=0, exact=False, nprod=3):
        self.name, self.kind, self.N, self.K, self.ring, self.make = name, kind, N, K, ring, make
        self.ldx, self.ld2, self.Nv, self.exact, self.nprod = ldx, ld2, Nv, exact, nprod

    def __repr__(self):
        return f"{self.name}-np{self.nprod}-N{self.N}-K{self.K}-ldx{self.ldx}-ld2{self.ld2}-Nv{self.Nv}"


def _rand(g, *shape):
    return torch.rand(*shape, generator=g, device="cuda")


def _randn(g, *shape):
    return torch.randn(*shape, generator=g, device="cuda")


def _stash(g, N, ldx, lo=0.0, hi=1.0):
    """[M_BIG + EXTRA][ldx] stash with zero padding (columns >= N)."""
    x = torch.zeros(M_BIG + EXTRA, ldx, device="cuda")
    x[:, :N] = lo + (hi - lo) * _rand(g, M_BIG + EXTRA, N)
    return x


def _nan(cols):
    return torch.full((M_BIG + EXTRA, cols), float("nan"), device="cuda")


def _relu_act(g, N, ldx):
    H = torch.zeros(M_BIG + EXTRA, ldx, device="cuda")
    H[:, :N] = torch.relu(_randn(g, M_BIG + EXTRA, N))
    return H


def _f32_out(OUT, M, N, ncols):
    """A ring-stored fp32 output of extent ncols: zeros in [N, ncols), the columns past it and rows >= M untouched."""
    assert not torch.isnan(OUT[:M, :ncols]).any() and torch.all(OUT[:M, N:ncols] == 0)
    assert torch.isnan(OUT[:M, ncols:]).all() and torch.isnan(OUT[M:]).all()


def _same_bits(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


def _chain_bwd(N, K, split):
    ldx = r8(N)
    ld2 = (256 if N == 217 else ldx) if split else ldx

    def make(g):
        D1, QT = _stash(g, N, ldx), _stash(g, N, ldx, -1.0, 1.0)
        Z, U = _nan(ldx), (_sentinel_split(M_BIG, ld2) if split else _nan(ldx))
        before, s = U.clone(), math.sqrt(0.5)

        def check(M, acc):
            z_ref, u_ref = _chain_bwd_ref(D1, QT, acc, s)
            ez = _check_f32(Z, M, N, z_ref)
            eu = _check_split(U, before, M, N, ldx, ld2, u_ref) if split else _check_f32(U, M, N, u_ref)
            return {"zbar": ez, "ubar": eu}
        return dict(X=D1, Y=QT, s=s, OUT=Z, OUT2=U), check
    return Case("chain_bwd_split" if split else "chain_bwd", 12 if split else 0, N, K, True, make, ldx, ld2, exact=True)


def _dgrad(N, K, sdf, split):
    ldx = r8(N)

    def make(g):
        D1 = _stash(g, N, ldx)
        ZB = _stash(g, N, ldx, -1.0, 1.0)
        ZB[M_BIG:] = 7.0
        zb0 = ZB.clone()
        sdfbar = _randn(g, M_BIG) if sdf else None
        wsdf = torch.zeros(ldx, device="cuda")
        wsdf[:N] = _randn(g, N)
        wsdf = wsdf if sdf else None
        OUT, Z16 = _nan(8), _sentinel_split(M_BIG, ldx)
        before, s, inv = Z16.clone(), 0.5, 1.0 / 3.0

        def check(M, acc):
            ref = _dgrad_ref(D1, zb0, acc, sdfbar, wsdf, M, N, s, inv)
            if split:
                e = _check_split(Z16, before, M, N, ldx, ldx, ref)
                assert _same_bits(ZB, zb0) and torch.isnan(OUT).all()
            else:
                e = _err(ZB[:M, :N], ref)
                assert e < BAR, e
                assert torch.all(ZB[:M, N:] == 0) and _same_bits(ZB[M:], zb0[M:])
            return {"zbar_prev": e}
        return dict(X=D1, Y=ZB, v1=sdfbar, v2=wsdf, s=s, s2=inv, OUT=OUT if split else None,
                    OUT2=Z16 if split else None), check
    kind = (14 if sdf else 13) if split else (2 if sdf else 1)
    return Case(f"dgrad{'_sdf' if sdf else ''}{'_split' if split else ''}", kind, N, K, True, make, ldx, ldx if split else 8,
                exact=True)


def _chain(Nv, E, K, split):
    ldx = max(r8(Nv), r8(E))

    def make(g):
        D1 = _stash(g, Nv, ldx)
        GE = _randn(g, M_BIG + EXTRA, ldx)
        ge0 = GE.clone()
        Q = _sentinel_split(M_BIG, ldx) if split else _nan(ldx)
        before, s = Q.clone(), math.sqrt(0.5)

        def check(M, acc):
            qt_ref, dge = _chain_ref(D1, acc, Nv, s)
            eq = _check_split(Q, before, M, Nv, ldx, ldx, qt_ref) if split else _check_f32(Q, M, Nv, qt_ref)
            errs = {"qt_prev": eq}
            if E:
                errs["ge"] = _err(GE[:M, :E], ge0[:M, :E].double() + dge)
                assert errs["ge"] < BAR, errs
            assert _same_bits(GE[:M, E:], ge0[:M, E:]) and _same_bits(GE[M:], ge0[M:])
            return errs
        if split:
            return dict(X=D1, s=s, OUT=GE, OUT2=Q), check
        return dict(X=D1, s=s, OUT=Q, OUT2=GE), check
    return Case("chain_split" if split else "chain", 15 if split else 3, Nv + E, K, True, make, ldx, ldx, Nv=Nv,
                exact=True)


def _dgrad_relu(N, K):
    ldx = r8(N)

    def make(g):
        H, OUT = _relu_act(g, N, ldx), _nan(ldx)

        def check(M, acc):
            e = _err(OUT[:M, :N], _relu_mask_ref(acc, H))
            assert e < BAR, e
            _f32_out(OUT, M, N, r4(N))
            return {"dgrad_relu": e}
        return dict(X=H, OUT=OUT), check
    return Case("dgrad_relu", 4, N, K, True, make, ldx, exact=True)


def _ge(N, K):
    ld2 = r8(N)

    def make(g):
        GE = _randn(g, M_BIG + EXTRA, ld2)
        ge0 = GE.clone()

        def check(M, acc):
            e = _err(GE[:M, :N], ge0[:M, :N].double() + acc)
            assert e < BAR, e
            assert _same_bits(GE[:M, N:], ge0[:M, N:]) and _same_bits(GE[M:], ge0[M:])
            return {"ge": e}
        return dict(X=torch.zeros(M_BIG, 8, device="cuda"), OUT=_nan(8), OUT2=GE), check
    return Case("ge", 5, N, K, True, make, 8, ld2)


def _stored(name, kind, N, K, ldx, ld2, ring, nprod=3):
    """The store-only functors: an fp32 OUT [ldx] and its bf16 split in OUT2 [2 ld2 bf16]."""
    bar = BAR if nprod == 3 else BAR_NP1

    def make(g):
        OUT, OUT2 = _nan(ldx), _sentinel_split(M_BIG, ld2)
        before = OUT2.clone()
        args = dict(X=torch.zeros(M_BIG, 8, device="cuda"), OUT=OUT, OUT2=OUT2)
        if kind == 6:
            bias = _randn(g, N) * 0.02
            D1 = _nan(ldx)
            if not ring:
                D1[:, N:] = 0.0      # the register path writes the padding only up to N rounded to 4
            args.update(Y=D1, v1=bias, s=0.7071067811865476)
        elif kind in (7, 8, 9):
            bias = _randn(g, N)
            args.update(v1=bias)
        if kind == 8:
            WxT = torch.zeros(6, ldx, device="cuda")
            WxT[:, :N] = _randn(g, 6, N)
            args.update(X=_randn(g, M_BIG, 8), v2=WxT)
        if kind == 11:
            args.update(X=_relu_act(g, N, ldx))

        def check(M, acc):
            errs = {}
            if kind == 6:
                out_ref, d1_ref = _value_ref(acc, bias, args["s"])
                errs["sp'"] = _err(D1[:M, :N], d1_ref)
                assert errs["sp'"] < BAR_D1, errs
                assert torch.all(D1[:M, N:] == 0) and torch.isnan(D1[M:, :N]).all()
            else:
                out_ref = {7: lambda: acc + bias.double()[None, :], 8: lambda: _color0_ref(acc, bias, args["X"], WxT),
                           9: lambda: torch.relu(acc + bias.double()[None, :]), 10: lambda: acc,
                           11: lambda: _relu_mask_ref(acc, args["X"])}[kind]()
            errs["out"] = _err(OUT[:M, :N], out_ref)
            assert errs["out"] < bar, errs
            ext = r4(N) if kind in (7, 10, 11) else N
            assert torch.all(OUT[:M, N:ext] == 0)
            _check_store(OUT, OUT2, before, M, ext, ext, ld2)
            return errs
        return args, check
    return Case(name, kind if nprod == 3 else kind + 100, N, K, ring, make, ldx, ld2, nprod=nprod)


def _plain(N, K, nprod):
    def make(g):
        Cm = torch.full((M_BIG + EXTRA, N), float("nan"), device="cuda")

        def check(M, acc):
            e = _err(Cm[:M], acc)
            assert e < BAR, e
            assert torch.isnan(Cm[M:]).all()
            return {"plain": e}
        return dict(OUT=Cm), check
    return Case("plain", "plain", N, K, _aligned(4 * N), make, nprod=nprod)


CASES = ([_chain_bwd(N, K, sp) for sp in (False, True) for _, N, K in SHAPES]
         + [_dgrad(N, K, sdf, sp) for sp in (False, True) for sdf in (False, True) for _, N, K in SHAPES]
         + [_chain(Nv, E, K, sp) for sp in (False, True) for _, Nv, E, K in CHAIN_SHAPES]
         + [_dgrad_relu(N, K) for _, N, K in SHAPES]
         + [_ge(N, K) for _, N, K in [(1000, 39, 256), (300, 64, 39), (129, 39, 39), (700, 39, 320)]]
         + [_stored("value", 6, N, K, ldx, ld2, _aligned(4 * N, 2 * N)) for _, N, K, ldx, ld2 in VALUE_SHAPES]
         + [_stored("bias", 7, N, K, r8(N), r8(N), _aligned(2 * r4(N))) for _, N, K in STORE_SHAPES]
         + [_stored(name, kind, N, K, r8(N), r8(N), ring(N), nprod) for nprod in (3, 1)
            for name, kind, shapes, ring in [("color0", 8, RELU_SHAPES, lambda n: False),
                                              ("relu", 9, RELU_SHAPES, lambda n: _aligned(2 * n)),
                                              ("store", 10, STORE_SHAPES, lambda n: _aligned(2 * r4(n))),
                                              ("dgrad_relu_split", 11, STORE_SHAPES, lambda n: _aligned(2 * r4(n)))]
            for _, N, K in shapes]
         + [_plain(N, K, nprod) for nprod in (3, 1) for _, N, K in [(1000, 64, 256), (300, 37, 39), (129, 128, 320),
                                                                      (513, 200, 64)]])


# ------------------------------------------------------------------------------------------------ the launches
def _lib():
    from avatarclip_b200 import _lib as L
    return L


def _launch(case, M, A, B, ws, args):
    L = _lib()
    lib = L.lib()
    vp, i32 = C.c_void_p, C.c_int32
    p = {k: (None if v is None else v.data_ptr()) for k, v in args.items() if isinstance(v, torch.Tensor) or v is None}
    if case.kind == "plain":
        f = lib.avc_tc_gemm_nt_test
        f.argtypes = [vp, vp, C.c_int64, i32, i32, i32, vp, vp, C.c_size_t, vp]
        f.restype = C.c_int
        L.check(f(A.data_ptr(), B.data_ptr(), M, case.N, case.K, case.nprod, p["OUT"], ws.data_ptr(), ws.numel(),
                  L.stream_ptr()), "avc_tc_gemm_nt_test")
    else:
        f = lib.avc_tc_epi_test
        f.argtypes = [i32, vp, vp, C.c_int64, i32, i32, i32, vp, vp, i32, vp, vp, C.c_float, C.c_float, vp, vp, i32, vp,
                      C.c_size_t, vp]
        f.restype = C.c_int
        L.check(f(case.kind, A.data_ptr(), B.data_ptr(), M, case.N, case.K, case.Nv, p.get("X"), p.get("Y"), case.ldx,
                  p.get("v1"), p.get("v2"), args.get("s", 1.0), args.get("s2", 1.0), p.get("OUT"), p.get("OUT2"),
                  case.ld2, ws.data_ptr(), ws.numel(), L.stream_ptr()), "avc_tc_epi_test")
    torch.cuda.synchronize()


def _hook(name, *argtypes):
    f = getattr(_lib().lib(), name)
    f.argtypes = list(argtypes)
    f.restype = C.c_int
    return f


@pytest.fixture
def set_cap():
    """avc_tc_nt_set_max_ctas, put back to no cap when the test ends, whatever happened."""
    f = _hook("avc_tc_nt_set_max_ctas", C.c_int32)
    yield f
    f(0)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=repr)
def test_persistent_epilogue(case, set_cap):
    last_grid, last_ring = _hook("avc_tc_nt_last_grid"), _hook("avc_tc_nt_last_ring")
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    g = torch.Generator(device="cuda").manual_seed(1000 + CASES.index(case))
    A = _randn(g, M_BIG, case.K)
    B = _randn(g, case.N, case.K) * 0.1
    ws = torch.empty(4 * (M_BIG + case.N) * r8(case.K) + 8 * M_BIG * max(case.ldx, case.ld2) + 8192, dtype=torch.uint8,
                     device="cuda")
    args, check = case.make(g)
    bufs = {k: v for k, v in args.items() if isinstance(v, torch.Tensor)}
    pristine = {k: v.clone() for k, v in bufs.items()}
    acc_big = A.double() @ B.double().t() if case.exact else _split_acc(A, B, case.nprod)
    tn = _tiles_n(case.N)
    leading = []
    for M, cap, claim in PLACEMENTS:
        for k, v in bufs.items():
            v.copy_(pristine[k])
        set_cap(cap * tn)
        try:
            _launch(case, M, A[:M], B, ws, args)
        finally:
            set_cap(0)
        grid, ring = last_grid(), last_ring()
        assert grid == _grid(M, case.N, sms, cap * tn), (grid, M, cap)
        lo, hi, ragged = _walk(M, case.N, grid)
        want = _claim(M, case.N, cap, claim)
        assert lo[0] >= want[0] and lo[1] >= want[1], (lo, want)
        assert ring == int(case.ring)
        errs = check(M, acc_big[:M])
        print(case, M, "cap", cap * tn, "grid", grid, "ring", ring, "tiles wg0", f"{lo[0]}-{hi[0]}", "wg1",
              f"{lo[1]}-{hi[1]}", "ragged on wg", ragged, " ".join(f"{k} {v:.3g}" for k, v in errs.items()))
        leading.append({k: v[:M_SMALL].clone() for k, v in bufs.items()})
    # bits do not depend on the placement: every run's first M_SMALL rows agree with the first
    for run, snap in enumerate(leading[1:], 1):
        for k, v in snap.items():
            assert _same_bits(v, leading[0][k]), (k, PLACEMENTS[run])


# ------------------------------------------------------------------------------------------------ coverage, no GPU
def test_coverage_claims():
    """What the placements above reach, from the grid rule, on the 132-SM and the 114-SM H100."""
    for sms in SMS:
        for case in CASES:
            ragged_wg = set()
            for M, cap, claim in PLACEMENTS:
                lo, _, ragged = _walk(M, case.N, _grid(M, case.N, sms, cap * _tiles_n(case.N)))
                want = _claim(M, case.N, cap, claim)
                assert lo[0] >= want[0] and lo[1] >= want[1], (sms, case, M, cap, lo)
                if M >= M_BENCH:      # every CTA's both warpgroups reach j >= 4
                    assert lo[0] >= 3 and lo[1] >= 3, (sms, case, M, lo)
                if cap:
                    ragged_wg.add(ragged)
            assert 1 in ragged_wg and 0 in ragged_wg, (sms, case)
    assert any(c.K > 256 for c in CASES)                                  # streamed B
    assert any(not c.ring for c in CASES)                                 # register stores
    assert any(not c.ring and c.kind == 8 for c in CASES)                 # EpiColor0
    assert any(not c.ring and c.N == 217 for c in CASES)                  # the skip layer's N = 217
    assert any(c.ldx == 224 and c.N == 200 for c in CASES)                # ring-stored zero padding
    assert {_tiles_n(c.N) for c in CASES} == {1, 2} and any(64 < c.N <= 128 for c in CASES)      # BN = 64 and 128
    assert {c.nprod for c in CASES} == {1, 3}
    kinds = {c.kind for c in CASES}
    assert kinds == set(range(16)) | {108, 109, 110, 111, "plain"}
