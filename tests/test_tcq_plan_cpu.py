"""Host logic of the small-M tensor-core kernel (gemm_tcq_kernel), checked without a GPU: the work cut that
b200awq_tcq_plan reports (the same function the launcher uses) must give every CTA a non-empty contiguous range, the
segments the kernel derives from a range (restated here exactly as the device code walks them) must cover every
(tile, k-step pair) exactly once, the per-tile ticket increments must add up to K / 128, and the tile-aligned cut must
never make a range straddle a tile."""
import ctypes

import pytest

from autoawq_b200._cabi import lib

SHAPES = [(4096, 4096), (4096, 6144), (4096, 14336), (4096, 28672), (14336, 4096), (8192, 1280), (1024, 8192),
          (8192, 7168), (3584, 8192), (512, 256), (1152, 384), (2048, 640), (128, 128), (4096, 128)]


def _plan(M, K, N, sms=132, mode=0, G=128):
    g, kp = ctypes.c_int(0), ctypes.c_int(0)
    rc = lib.b200awq_tcq_plan(M, K, N, G, sms, mode, ctypes.byref(g), ctypes.byref(kp))
    return rc, g.value, kp.value


def _segments(t_begin, t_end, KP):
    """(tile, first pair, last pair + 1) of a CTA's range: the loop every warp role of the kernel runs."""
    t, out = t_begin, []
    while t < t_end:
        nt = t // KP
        d0 = t - nt * KP
        d1 = KP if KP - d0 < t_end - t else d0 + (t_end - t)
        out.append((nt, d0, d1))
        t += d1 - d0
    return out


@pytest.mark.parametrize("K,N", SHAPES)
@pytest.mark.parametrize("M", [1, 5, 16, 63, 64, 128])
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_plan_covers_every_pair_once(K, N, M, mode):
    rc, grid, KP = _plan(M, K, N, mode=mode)
    assert rc == 0 and KP == K // 128
    n_tiles = N // 128
    T = n_tiles * KP
    assert 1 <= grid <= 132
    seen = [[0] * KP for _ in range(n_tiles)]
    tickets = [0] * n_tiles
    for b in range(grid):
        t0, t1 = T * b // grid, T * (b + 1) // grid
        assert t1 > t0, "a CTA without work would deadlock nothing but wastes an SM: the launcher must not create it"
        segs = _segments(t0, t1, KP)
        assert len(segs) <= 2 + (t1 - t0) // KP
        for nt, d0, d1 in segs:
            assert 0 <= d0 < d1 <= KP
            for d in range(d0, d1):
                seen[nt][d] += 1
            if not (d0 == 0 and d1 == KP):      # partial segment: split-K ticket
                tickets[nt] += d1 - d0
        if mode == 2 or (mode == 0 and (n_tiles <= 132 or M >= 64)):
            if n_tiles <= 132 or n_tiles % -(-n_tiles // 132) == 0:
                assert len({nt for nt, _, _ in segs}) == len(segs), "one segment per tile"
                if n_tiles <= 132:
                    assert len(segs) == 1, "tile-aligned cut: a range never straddles a tile"
    assert all(c == 1 for row in seen for c in row)
    assert all(t in (0, KP) for t in tickets), "partial segments of a tile complete exactly K / 128"


def test_plan_envelope_and_errors():
    assert _plan(129, 4096, 4096)[0] != 0          # M above the kernel's range
    assert _plan(16, 4096 + 64, 4096)[0] != 0      # K % 128
    assert _plan(16, 4096, 4096 + 64)[0] != 0      # N % 128
    assert _plan(16, 4096, 4096, G=32)[0] != 0     # G < 64
    assert _plan(16, 4096, 4096, G=64)[0] == 0
    assert lib.b200awq_tcq_plan(16, 4096, 4096, 128, 132, 0, None, None) != 0


def test_plan_examples_from_design():
    """The cuts DESIGN 3.3b quotes: 112 whole tiles for 4096 x 14336, 4 ranges per tile for 4096 x 4096, balanced 132
    below 64 tokens and 112 x 2 tiles from 64 tokens on 4096 x 28672."""
    assert _plan(16, 4096, 14336)[1] == 112
    assert _plan(16, 4096, 4096)[1] == 128
    assert _plan(16, 4096, 28672)[1] == 132
    assert _plan(64, 4096, 28672)[1] == 112
    assert _plan(16, 4096, 6144)[1] == 96
