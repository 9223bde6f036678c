"""Column / row sharding of packed AWQ tensors across the GPUs of one box (SURVEY.md 8e).

The reference has no tensor parallelism (multi-GPU = accelerate layer placement, awq/models/base.py:527-535);
BASELINE config 5 (Llama-3-70B on 8 x H100) needs it.  A linear is independent per output column and
additive over K, and the packed formats slice cleanly:

  column-parallel (split N; qkv / gate / up):  GEMM layout  qweight[:, n0/8:n1/8], qzeros[:, n0/8:n1/8],
      scales[:, n0:n1]  with n0, n1 multiples of 8 - the same legality argument as fuse_qkv's concatenation
      (awq/utils/fused_utils.py:87-96).  No collective: the consumer (attention / SiLU*mul) is local in N.
  row-parallel (split K; o / down):  qweight[k0:k1, :], qzeros[k0/G:k1/G, :], scales[k0/G:k1/G, :] with
      k0, k1 multiples of G.  Each rank produces a partial [M, N]; ONE all-reduce (NCCL over NVLink, fp16
      output) per attention block and one per MLP block finishes it.

One process per GPU; the collective is torch.distributed (NCCL on GPUs, gloo in the CPU tests).
"""
from __future__ import annotations

from dataclasses import dataclass

import torch


def _bounds(total: int, rank: int, world: int, quantum: int):
    """Contiguous [lo, hi) share of `total` for `rank`, in units of `quantum`."""
    if total % quantum != 0:
        raise ValueError(f"{total} is not a multiple of {quantum}")
    units = total // quantum
    lo = units * rank // world
    hi = units * (rank + 1) // world
    return lo * quantum, hi * quantum


@dataclass
class PackedGemm:
    qweight: torch.Tensor  # [K, N/8] int32
    qzeros: torch.Tensor   # [K/G, N/8] int32
    scales: torch.Tensor   # [K/G, N] fp16
    bias: torch.Tensor | None = None

    @property
    def in_features(self):
        return self.qweight.shape[0]

    @property
    def out_features(self):
        return self.qweight.shape[1] * 8

    @property
    def group_size(self):
        return self.qweight.shape[0] // self.scales.shape[0]


def shard_columns(p: PackedGemm, rank: int, world: int, quantum: int = 8) -> PackedGemm:
    """Column-parallel slice (split N on `quantum`-column boundaries, quantum % 8 == 0)."""
    if quantum % 8 != 0:
        raise ValueError("column quantum must be a multiple of 8 (one packed word)")
    n0, n1 = _bounds(p.out_features, rank, world, quantum)
    return PackedGemm(
        p.qweight[:, n0 // 8 : n1 // 8].contiguous(),
        p.qzeros[:, n0 // 8 : n1 // 8].contiguous(),
        p.scales[:, n0:n1].contiguous(),
        None if p.bias is None else p.bias[n0:n1].contiguous(),
    )


def shard_rows(p: PackedGemm, rank: int, world: int) -> PackedGemm:
    """Row-parallel slice (split K on group boundaries).  The bias is kept on rank 0 only so that the
    all-reduce adds it exactly once."""
    G = p.group_size
    k0, k1 = _bounds(p.in_features, rank, world, G)
    return PackedGemm(
        p.qweight[k0:k1].contiguous(),
        p.qzeros[k0 // G : k1 // G].contiguous(),
        p.scales[k0 // G : k1 // G].contiguous(),
        p.bias if (p.bias is not None and rank == 0) else None,
    )


def shard_qkv(p: PackedGemm, n_heads: int, n_kv_heads: int, head_dim: int, rank: int, world: int) -> PackedGemm:
    """Fused qkv (columns = [q heads | k heads | v heads], awq/utils/fused_utils.py:67-74) split by head
    group so attention stays local: rank r gets q heads [r*H/W, (r+1)*H/W) and the matching kv heads."""
    if n_heads % world or n_kv_heads % world:
        raise ValueError("heads must divide evenly across ranks")
    qn, kvn = n_heads * head_dim, n_kv_heads * head_dim
    parts = []
    for base, width in ((0, qn), (qn, kvn), (qn + kvn, kvn)):
        lo, hi = _bounds(width, rank, world, head_dim)
        parts.append((base + lo, base + hi))
    cols = [slice(a // 8, b // 8) for a, b in parts]
    return PackedGemm(
        torch.cat([p.qweight[:, c] for c in cols], dim=1).contiguous(),
        torch.cat([p.qzeros[:, c] for c in cols], dim=1).contiguous(),
        torch.cat([p.scales[:, a:b] for a, b in parts], dim=1).contiguous(),
        None if p.bias is None else torch.cat([p.bias[a:b] for a, b in parts]).contiguous(),
    )


def x_slice_for_rows(x: torch.Tensor, in_features: int, group_size: int, rank: int, world: int) -> torch.Tensor:
    """The activation columns a row-parallel shard consumes (the column-parallel producer already left
    exactly these on this rank when both use the same `world` and group-aligned split)."""
    k0, k1 = _bounds(in_features, rank, world, group_size)
    return x[..., k0:k1]


def all_reduce_sum(y: torch.Tensor, group=None) -> torch.Tensor:
    """The single collective of a column->row pair: sum of the partial outputs (in place)."""
    import torch.distributed as dist

    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(y, op=dist.ReduceOp.SUM, group=group)
    return y


class TensorParallelMLP:
    """gate|up (column-parallel, fused) -> SiLU*mul -> down (row-parallel) -> all-reduce, on this repository's kernels.
    Per-rank weights are the slices above; used by the 70B-shape tensor-parallel bench leg (bench.py `tp70b`) and
    the tests.  gate / up are split on the boundaries of down's K split (its group size), so the activation width
    of a rank always equals its number of down rows, also when (I / G) % world != 0."""

    def __init__(self, gate: PackedGemm, up: PackedGemm, down: PackedGemm, rank: int, world: int, group=None,
                 all_reduce=None):
        """`all_reduce`: callable summing a tensor over the ranks in place (e.g. autoawq_b200.comm.OneShotAllReduce);
        default: torch.distributed.all_reduce (NCCL on GPUs, gloo in the CPU tests)."""
        from . import ext

        self.ext, self.group, self.all_reduce = ext, group, all_reduce
        quantum = max(8, down.group_size)
        g, u = shard_columns(gate, rank, world, quantum), shard_columns(up, rank, world, quantum)
        bias = None
        if g.bias is not None or u.bias is not None:
            z = lambda p: p.bias if p.bias is not None else torch.zeros(  # noqa: E731
                p.out_features, dtype=torch.float16, device=p.qweight.device)
            bias = torch.cat([z(g), z(u)]).contiguous()
        self.gu = PackedGemm(torch.cat([g.qweight, u.qweight], 1).contiguous(),
                             torch.cat([g.qzeros, u.qzeros], 1).contiguous(),
                             torch.cat([g.scales, u.scales], 1).contiguous(), bias)
        self.down = shard_rows(down, rank, world)
        if g.out_features != self.down.in_features or u.out_features != self.down.in_features:
            raise ValueError(f"rank {rank}/{world}: gate/up shard width {g.out_features}/{u.out_features} != down shard "
                             f"rows {self.down.in_features}")

    def __call__(self, x: torch.Tensor) -> torch.Tensor:
        e = self.ext
        gu = e.linear_forward("gemm", x, self.gu.qweight, self.gu.scales, self.gu.qzeros, self.gu.group_size,
                              self.gu.bias)
        act = torch.empty((gu.shape[0], gu.shape[1] // 2), dtype=torch.float16, device=gu.device)
        e.silu_and_mul(act, gu)
        y = e.linear_forward("gemm", act, self.down.qweight, self.down.scales, self.down.qzeros, self.down.group_size,
                             self.down.bias)
        return self.all_reduce(y) if self.all_reduce is not None else all_reduce_sum(y, self.group)
