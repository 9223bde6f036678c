"""Tile list of the grouped tensor-core kernel (moe_tc_kernel), checked without a GPU.  b200awq_moe_tc_plan walks a host
copy of expert_ids with the function the kernel's warp roles enumerate through; on random and adversarial routings
every sorted position must be covered exactly once per 128-column tile, no tile may span two experts or exceed the
token tile, and the token tiles of one (expert, column tile) must be adjacent (CTAs that run together then share the
expert's weight slab in L2).  The kernel's register / spill budget comes from ptxas."""
import ctypes

import numpy as np
import pytest

from _toolchain import entries, needs_nvcc
from autoawq_b200._cabi import lib
from oracle import awq_oracle as O

BLOCK = 16


def _plan(expert_ids, n_blocks, E, N, BT, block=BLOCK, max_tiles=1 << 16):
    ids = np.ascontiguousarray(expert_ids, dtype=np.int32)
    out = np.full((max_tiles, 4), -7, dtype=np.int32)
    n = ctypes.c_int(-1)
    rc = lib.b200awq_moe_tc_plan(ids.ctypes.data, n_blocks, block, E, N, BT, 132, out.ctypes.data, max_tiles,
                                 ctypes.byref(n))
    return rc, out[:max(0, min(n.value, max_tiles))], n.value


def _routing(kind, rng):
    """topk_ids [T, topk] and E for one named routing."""
    if kind == "random-mixtral":
        return np.stack([rng.permutation(8)[:2] for _ in range(700)]), 8
    if kind == "one-expert":                     # every token on expert 5
        return np.full((333, 1), 5), 8
    if kind == "two-of-eight":                   # experts 0, 1, 2, 4, 5, 7 have no token
        return np.tile(np.array([[3, 6]]), (190, 1)), 8
    if kind == "runs-of-one":                    # every expert gets exactly one slot
        return np.arange(8).reshape(4, 2), 8
    if kind == "runs-of-exactly-bt":             # 128 slots each: one full tile at BT = 128, two at 64, four at 32
        return np.repeat(np.arange(8), 128).reshape(-1, 2), 8
    if kind == "bt-plus-one":                    # a run one longer than every token tile
        return np.concatenate([np.full(129, 2), np.full(33, 4), np.full(65, 6)]).reshape(-1, 1), 8
    if kind == "e64-top6":
        return np.stack([rng.permutation(64)[:6] for _ in range(257)]), 64
    raise AssertionError(kind)


KINDS = ["random-mixtral", "one-expert", "two-of-eight", "runs-of-one", "runs-of-exactly-bt", "bt-plus-one", "e64-top6"]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("BT", [32, 64, 128])
@pytest.mark.parametrize("N", [96, 512, 28672])
def test_tiles_cover_every_sorted_position_once(kind, BT, N):
    rng = np.random.default_rng(len(kind) * 1000 + BT + N)
    topk_ids, E = _routing(kind, rng)
    _, expert_ids, npost = O.moe_align_block_size(topk_ids, BLOCK, E)
    n_blocks = npost // BLOCK
    rc, tiles, n = _plan(expert_ids, n_blocks, E, N, BT)
    assert rc == 0 and n == len(tiles) > 0
    n_tiles = -(-N // 128)
    covered = np.zeros((n_tiles, npost), dtype=np.int32)
    for e, pos0, rows, nt in tiles:
        assert 1 <= rows <= BT and 0 <= nt < n_tiles and 0 <= pos0 and pos0 + rows <= npost
        blocks = expert_ids[pos0 // BLOCK:(pos0 + rows - 1) // BLOCK + 1]
        assert (blocks == e).all(), "a tile spans two experts, or names the wrong one"
        covered[nt, pos0:pos0 + rows] += 1
    assert (covered == 1).all(), "a sorted position is missed or covered twice"
    # token tiles of one (expert, column tile) are adjacent, in ascending position, and only the last is partial
    keys = [(int(e), int(nt)) for e, _, _, nt in tiles]
    groups = [k for i, k in enumerate(keys) if i == 0 or keys[i - 1] != k]
    assert len(groups) == len(set(groups)), "an (expert, column tile) group is split"
    for i in range(1, len(tiles)):
        if keys[i] == keys[i - 1]:
            assert tiles[i - 1][2] == BT and tiles[i][1] == tiles[i - 1][1] + BT
    # exactly the experts that have tokens appear
    assert {k[0] for k in keys} == set(np.unique(topk_ids).tolist())


def test_tile_count_examples():
    """Mixtral prefill, 4096 tokens top-2 spread evenly: 8 experts x 1024 slots -> 8 token tiles of 128 x 224 column
    tiles (gate|up, N = 28672)."""
    topk_ids = np.stack([(np.arange(4096) % 8), ((np.arange(4096) + 1) % 8)], axis=1)
    _, expert_ids, npost = O.moe_align_block_size(topk_ids, BLOCK, 8)
    rc, tiles, n = _plan(expert_ids, npost // BLOCK, 8, 28672, 128)
    assert rc == 0 and n == 8 * 8 * 224
    assert tiles[0].tolist() == [0, 0, 128, 0] and tiles[8].tolist() == [0, 0, 128, 1]
    # truncated output buffer: the count is still the full one, nothing is written past max_tiles
    rc, tiles, n = _plan(expert_ids, npost // BLOCK, 8, 28672, 128, max_tiles=10)
    assert rc == 0 and n == 8 * 8 * 224 and len(tiles) == 10


def test_block_size_larger_than_token_tile():
    """block_size 64 with BT = 32: a block is two token tiles; a run of one slot still covers its whole padded block."""
    topk_ids = np.array([[0], [2], [2]])
    _, expert_ids, npost = O.moe_align_block_size(topk_ids, 64, 4)
    rc, tiles, n = _plan(expert_ids, npost // 64, 4, 128, 32, block=64)
    assert rc == 0 and tiles.tolist() == [[0, 0, 32, 0], [0, 32, 32, 0], [2, 64, 32, 0], [2, 96, 32, 0]]


def test_out_of_range_expert_has_no_tiles_and_empty_list():
    rc, tiles, n = _plan([0, 0, 9, -1, 3], 5, 8, 256, 32)
    assert rc == 0 and sorted({int(t[0]) for t in tiles}) == [0, 3]
    assert _plan([0], 0, 8, 256, 32)[2] == 0


def test_plan_argument_errors():
    ids = np.zeros(4, dtype=np.int32)
    out = np.zeros((4, 4), dtype=np.int32)
    n = ctypes.c_int(0)
    ok = lambda **kw: lib.b200awq_moe_tc_plan(  # noqa: E731
        kw.get("ids", ids.ctypes.data), 4, kw.get("block", 16), kw.get("E", 8), kw.get("N", 256), kw.get("BT", 64),
        kw.get("sms", 132), out.ctypes.data, 4, ctypes.byref(n))
    assert ok() == 0
    assert ok(ids=None) != 0 and ok(BT=48) != 0 and ok(N=100) != 0 and ok(sms=0) != 0
    assert ok(block=8) != 0 and ok(E=257) != 0


@needs_nvcc
def test_moe_tc_kernel_register_and_spill_budget():
    """One CTA of 512 threads per SM, accumulators in the consumer warpgroups' registers: registers x 512 must fit the
    64 K register file and nothing may spill."""
    found = entries("gemm_tc.cu", r"moe_tc_kernel")
    assert len(found) == 6, found          # BT in {32, 64, 128} x 1 or 2 quantisation groups per k-step
    for name, (regs, stack, st, ld) in found.items():
        assert st == 0 and ld == 0 and stack == 0, f"{name}: spills"
        assert regs * 512 <= 65536, f"{name}: {regs} registers x 512 threads"
