"""Placement independence of the fused SDF value-chain kernel (k_sdf_chain, csrc/avc_chain.cu) under its tile schedule:
64-point tiles dealt over the CTAs first (tile t on CTA t % grid), a CTA's tiles alternating between its two consumer
warpgroups, which take strict turns at the tensor pipe layer by layer.

Through kind 27 of avc_neus_kernel_test (as in test_neus_value_chain_gpu.py), at tile counts around one and two tiles
per SM (SMs - 1, SMs, SMs + 1, 2 SMs, 2 SMs + 1: on a 132-SM H100 131, 132, 133, 264 and 265 tiles, so CTA 0 gets a
second tile on warpgroup 1 and then a third, alone, on warpgroup 0), at 1 and 2 tiles, with a ragged last tile on either
warpgroup, and with the grid capped by the test hook avc_chain_set_max_ctas at 1, 2 and 3 CTAs, so that one CTA walks
every tile, odd and even counts of them, alternating between its warpgroups.  At every placement each point's sdf must
have the bits of the same point evaluated in a launch of its own (launches of 50 points: one CTA, warpgroup 0, rows
that do not line up with the 64-point tiles), and meet the fp64 bar of test_neus_value_chain_gpu.py.  The networks:
bench.py's (8 hidden linears, the skip concat inside), one hidden linear (one MMA step per tile, so the turn passes at
every tile) and 4 hidden linears with partial last k-blocks."""
import ctypes as C

import pytest
import torch

import test_neus_chain_kernels_gpu as K
import test_neus_value_chain_gpu as V

pytestmark = pytest.mark.gpu

ALONE = 50          # points per launch of the reference runs
NAMES = ["b2", "l1", "w80"]


def _hook(name, *argtypes):
    from avatarclip_b200 import _lib
    f = getattr(_lib.lib(), name)
    f.argtypes = list(argtypes)
    f.restype = C.c_int
    return f


class _Cap:
    """avc_chain_set_max_ctas for the duration of a with-block, put back to no cap whatever happens."""

    def __init__(self, n):
        self.n = n
        self.f = _hook("avc_chain_set_max_ctas", C.c_int32)

    def __enter__(self):
        self.f(self.n)

    def __exit__(self, *exc):
        self.f(0)


def _last_grid():
    return _hook("avc_chain_last_grid")()


_CASES = {}


def _case(name):
    """The configuration at 2 SMs + 1 tiles of 64 points: the encoded pairs, the output of launches of ALONE points each,
    the fp64 reference and its bar."""
    if name not in _CASES:
        net = V._net(name)
        P = 64 * (2 * V._sms() + 1)
        p0, ps = net.encode(V._points(P, 21))
        alone = torch.empty(P, dtype=torch.float32, device="cuda")
        for r in range(0, P, ALONE):
            n = min(ALONE, P - r)
            out = net.run(p0[r:r + n], None if ps is None else ps[r:r + n], n)
            assert out.intact()
            assert _last_grid() == 1
            alone[r:r + n] = out.t
        ref = net.reference(p0, ps, P)
        twin = net.reference(p0, ps, P, dtype=torch.float32, split_acts=True)
        _CASES[name] = (net, p0, ps, alone, ref, K._bar(ref, twin, V.FLOOR))
    return _CASES[name]


def _check(name, P, cap, grid):
    net, p0, ps, alone, ref, bar = _case(name)
    if cap:
        with _Cap(cap):
            out = net.run(p0, ps, P)
    else:
        out = net.run(p0, ps, P)
    assert out.intact()
    assert _last_grid() == grid, (_last_grid(), grid)
    e = (out.t.double() - ref[:P]).abs().max().item() / ref.abs().max().item()
    print(f"[worst] value_chain {name} P {P} cap {cap} grid {grid} err {e:.2e} bar {bar:.1e}")
    assert e <= bar, (name, P, cap, e, bar)
    assert torch.equal(V._bits(out.t), V._bits(alone[:P])), (name, P, cap)


# tiles, rows short of whole tiles; "s" stands for the number of SMs
TILES = [(1, 0), (2, 0), ("s-1", 0), ("s", 0), ("s+1", 0), ("2s", 0), ("2s+1", 0),
         (1, 23),            # one ragged tile
         ("s", 23),          # ragged last tile on warpgroup 0 of the last CTA
         ("s+1", 23),        # ragged last tile on warpgroup 1 of CTA 0
         ("2s+1", 23)]       # ragged third tile of CTA 0, on warpgroup 0 alone


@pytest.mark.parametrize("tiles,short", TILES)
@pytest.mark.parametrize("name", NAMES)
def test_natural_grid(name, tiles, short):
    """One CTA per SM at most, never more CTAs than tiles."""
    s = V._sms()
    T = tiles if isinstance(tiles, int) else {"s-1": s - 1, "s": s, "s+1": s + 1, "2s": 2 * s, "2s+1": 2 * s + 1}[tiles]
    _check(name, 64 * T - short, 0, min(T, s))


# (cap, tiles, rows short): at cap 1 CTA 0 walks every tile (11: 6 on warpgroup 0 with the ragged last one, 5 on
# warpgroup 1); at 2 the ragged tile 10 is CTA 0's sixth, on warpgroup 1; at 3 CTA 2 has an odd count (3) and CTA 1 the
# ragged tile on warpgroup 1
CAPS = [(1, 1, 0), (1, 2, 0), (1, 3, 0), (1, 11, 23), (1, 40, 0), (2, 11, 23), (2, 3, 0), (3, 11, 23), (3, 12, 0)]


@pytest.mark.parametrize("cap,tiles,short", CAPS)
@pytest.mark.parametrize("name", NAMES)
def test_capped_grid(name, cap, tiles, short):
    _check(name, 64 * tiles - short, cap, min(cap, tiles))


def test_cap_hook_returns_previous():
    f = _hook("avc_chain_set_max_ctas", C.c_int32)
    try:
        assert f(5) == 0
        assert f(-3) == 5
        assert f(0) == 0
    finally:
        f(0)
