"""Checkpoint -> (sharded) packed device buffers, without accelerate (SURVEY.md 8f #4).

The reference loads an AWQ checkpoint by building the whole module tree on the meta device and letting accelerate's
`load_checkpoint_and_dispatch` place every tensor (awq/models/base.py:505-535); multi-GPU there means layer placement,
every rank would read every tensor.  For the tensor-parallel decode of BASELINE config 5 each rank needs only its
column / row slice of every packed tensor (autoawq_b200/shard.py): this loader reads exactly those bytes.  safetensors
files are memory-mapped and sliceable, so a column shard `qweight[:, a:b]` or a row shard `qweight[k0:k1]` is read
straight from the file into the rank's device buffer.

Tensor names follow the reference's module buffers (awq/modules/linear/gemm.py:135-170): `<prefix>.qweight`,
`<prefix>.qzeros`, `<prefix>.scales`, optional `<prefix>.bias`, GEMM layout (the checkpoint default,
awq/models/_config.py:14).
"""
from __future__ import annotations

import json
import os
from typing import Dict, Iterable, Optional

import torch

from .shard import PackedGemm, _bounds

# which way a linear is split, by the last component of its name (Llama / Mistral / Mixtral / Qwen naming)
COLUMN_PARALLEL = ("q_proj", "k_proj", "v_proj", "gate_proj", "up_proj", "w1", "w3", "qkv_proj", "gate_up_proj")
ROW_PARALLEL = ("o_proj", "down_proj", "w2", "dense", "out_proj")
# (the fused names qkv_proj / gate_up_proj are split PER SECTION, see column_sections: one contiguous N range would
# leave rank 0 with q heads only / gate columns only)


class CheckpointIndex:
    """name -> file for a directory of *.safetensors shards (uses model.safetensors.index.json when present)."""

    def __init__(self, path: str):
        self.files: Dict[str, str] = {}
        if os.path.isfile(path):
            self._scan(path)
            return
        idx = os.path.join(path, "model.safetensors.index.json")
        if os.path.exists(idx):
            with open(idx) as f:
                wm = json.load(f)["weight_map"]
            self.files = {k: os.path.join(path, v) for k, v in wm.items()}
        else:
            for fn in sorted(os.listdir(path)):
                if fn.endswith(".safetensors"):
                    self._scan(os.path.join(path, fn))
        if not self.files:
            raise FileNotFoundError(f"no safetensors tensors under {path}")

    def _scan(self, file: str):
        from safetensors import safe_open

        with safe_open(file, framework="pt", device="cpu") as f:
            for k in f.keys():
                self.files[k] = file

    def linear_prefixes(self) -> list:
        """Prefixes that hold a complete packed linear (qweight + qzeros + scales)."""
        out = []
        for k in self.files:
            if k.endswith(".qweight"):
                p = k[: -len(".qweight")]
                if p + ".qzeros" in self.files and p + ".scales" in self.files:
                    out.append(p)
        return sorted(out)


def split_mode(prefix: str, column: Iterable[str] = COLUMN_PARALLEL, row: Iterable[str] = ROW_PARALLEL) -> str:
    leaf = prefix.rsplit(".", 1)[-1]
    if leaf in column:
        return "column"
    if leaf in row:
        return "row"
    return "replicate"


def _read(index: CheckpointIndex, name: str, device, rows: Optional[slice] = None, cols: Optional[slice] = None):
    from safetensors import safe_open

    with safe_open(index.files[name], framework="pt", device="cpu") as f:
        sl = f.get_slice(name)
        nd = len(sl.get_shape())
        if nd == 1:
            t = sl[cols] if cols is not None else sl[:]
        else:
            t = sl[rows if rows is not None else slice(None), cols if cols is not None else slice(None)]
    return t.contiguous().to(device, non_blocking=False)


def column_sections(prefix: str, N: int, sections=None, qkv_heads=None):
    """[(start, width, quantum or None)] of a column-parallel tensor.  Plain projections are one section; the fused
    names need their section widths: gate_up_proj = two halves; qkv_proj = (n_heads, n_kv_heads, head_dim) ->
    q | k | v split by head (quantum = head_dim so attention stays local, as shard.shard_qkv does)."""
    leaf = prefix.rsplit(".", 1)[-1]
    if sections is not None:
        out, base = [], 0
        for w in sections:
            out.append((base, int(w), None))
            base += int(w)
        if base != N:
            raise ValueError(f"{prefix}: sections {list(sections)} do not add up to N = {N}")
        return out
    if leaf == "gate_up_proj":
        if N % 2:
            raise ValueError(f"{prefix}: odd width {N} cannot be [gate | up]")
        return [(0, N // 2, None), (N // 2, N // 2, None)]
    if leaf == "qkv_proj":
        if qkv_heads is None:
            raise ValueError(f"{prefix}: a fused qkv tensor needs qkv_heads=(n_heads, n_kv_heads, head_dim) to be "
                             "split by head; a contiguous column range would give a rank q heads only")
        h, hkv, d = qkv_heads
        if (h + 2 * hkv) * d != N:
            raise ValueError(f"{prefix}: qkv_heads {qkv_heads} do not match N = {N}")
        return [(0, h * d, d), (h * d, hkv * d, d), ((h + hkv) * d, hkv * d, d)]
    return [(0, N, None)]


def load_packed_linear(index: CheckpointIndex, prefix: str, device, tp_rank: int = 0, tp_world: int = 1,
                       mode: Optional[str] = None, column_quantum: Optional[int] = None, sections=None,
                       qkv_heads=None) -> PackedGemm:
    """One packed linear, or this rank's shard of it.  mode: "column" (split N), "row" (split K on group
    boundaries; the bias stays on rank 0 so the all-reduce adds it once), "replicate", or None = by name
    (`split_mode`).

    Column quantum: a column-parallel linear feeds a row-parallel one (gate/up -> down, q/k/v -> attention -> o)
    whose K is split on ITS group boundaries, so the producer's columns must be split on the same boundaries or
    the shards do not line up whenever (N / G) % tp_world != 0 (e.g. I = 11008, G = 128, tp = 4: columns from
    2752 but rows from 2688).  Default = this linear's own group size (the model-wide q_group_size,
    awq/models/_config.py:12), never less than one packed word (8); k_proj / v_proj feed attention, not a
    row-parallel K split, and default to one packed word (pass head_dim to keep heads whole); pass the consumer's
    group size / head_dim when they differ.  Fused tensors are split per section (`column_sections`)."""
    from safetensors import safe_open

    mode = mode or split_mode(prefix)
    if tp_world == 1:
        mode = "replicate"
    with safe_open(index.files[prefix + ".qweight"], framework="pt", device="cpu") as f:
        K, NW = f.get_slice(prefix + ".qweight").get_shape()
    with safe_open(index.files[prefix + ".scales"], framework="pt", device="cpu") as f:
        KG, N = f.get_slice(prefix + ".scales").get_shape()
    if N != NW * 8 or K % KG != 0:
        raise ValueError(f"{prefix}: qweight {K}x{NW} and scales {KG}x{N} do not form a GEMM-layout linear")
    G = K // KG
    has_bias = prefix + ".bias" in index.files
    if mode == "column":
        parts = []
        for base, width, q in column_sections(prefix, N, sections, qkv_heads):
            kv = prefix.rsplit(".", 1)[-1] in ("k_proj", "v_proj")
            quantum = column_quantum if column_quantum is not None else (q if q is not None else (8 if kv else max(8, G)))
            if quantum % 8 != 0:
                raise ValueError("column quantum must be a multiple of 8 (one packed word)")
            if width % quantum != 0:
                raise ValueError(f"{prefix}: section width {width} is not a multiple of the column quantum {quantum}")
            n0, n1 = _bounds(width, tp_rank, tp_world, quantum)
            n0, n1 = base + n0, base + n1
            cw = slice(n0 // 8, n1 // 8)
            parts.append(PackedGemm(_read(index, prefix + ".qweight", device, cols=cw),
                                    _read(index, prefix + ".qzeros", device, cols=cw),
                                    _read(index, prefix + ".scales", device, cols=slice(n0, n1)),
                                    _read(index, prefix + ".bias", device, cols=slice(n0, n1)) if has_bias else None))
        return parts[0] if len(parts) == 1 else fuse_columns(parts)
    if mode == "row":
        k0, k1 = _bounds(K, tp_rank, tp_world, G)
        return PackedGemm(_read(index, prefix + ".qweight", device, rows=slice(k0, k1)),
                          _read(index, prefix + ".qzeros", device, rows=slice(k0 // G, k1 // G)),
                          _read(index, prefix + ".scales", device, rows=slice(k0 // G, k1 // G)),
                          _read(index, prefix + ".bias", device) if (has_bias and tp_rank == 0) else None)
    if mode != "replicate":
        raise ValueError(mode)
    return PackedGemm(_read(index, prefix + ".qweight", device), _read(index, prefix + ".qzeros", device),
                      _read(index, prefix + ".scales", device),
                      _read(index, prefix + ".bias", device) if has_bias else None)


def load_packed_linears(path: str, device, tp_rank: int = 0, tp_world: int = 1, prefixes: Optional[Iterable[str]] = None,
                        column_quantum: Optional[int] = None, qkv_heads=None) -> Dict[str, PackedGemm]:
    """Every packed linear of a checkpoint directory (or the given prefixes), sharded for (tp_rank, tp_world).
    q/k/v projections (and a fused qkv_proj) are split by head when `qkv_heads=(n_heads, n_kv_heads, head_dim)` is
    given; everything column-parallel otherwise on group boundaries (see load_packed_linear)."""
    index = CheckpointIndex(path)
    out = {}
    for p in (list(prefixes) if prefixes is not None else index.linear_prefixes()):
        cq = column_quantum
        if cq is None and qkv_heads is not None and p.rsplit(".", 1)[-1] in ("q_proj", "k_proj", "v_proj"):
            cq = qkv_heads[2]
        out[p] = load_packed_linear(index, p, device, tp_rank, tp_world, None, cq, qkv_heads=qkv_heads)
    check_tp_alignment(out, tp_rank, tp_world)
    return out


def check_tp_alignment(shards: Dict[str, PackedGemm], tp_rank: int, tp_world: int) -> None:
    """Column-parallel producers and the row-parallel consumer of the same block must hold matching widths on every
    rank: gate/up (w1/w3) columns == down (w2) rows.  Raises instead of letting a caller pair the wrong channels."""
    if tp_world == 1:
        return
    by_parent: Dict[str, Dict[str, PackedGemm]] = {}
    for name, p in shards.items():
        parent, leaf = name.rsplit(".", 1) if "." in name else ("", name)
        by_parent.setdefault(parent, {})[leaf] = p
    for parent, d in by_parent.items():
        for prods, cons in ((("gate_proj", "up_proj"), "down_proj"), (("w1", "w3"), "w2")):
            if cons in d:
                for pr in prods:
                    if pr in d and d[pr].out_features != d[cons].in_features:
                        raise ValueError(f"{parent}: rank {tp_rank}/{tp_world} holds {d[pr].out_features} columns of {pr} "
                                         f"but {d[cons].in_features} rows of {cons}; split both on the same boundaries")
        if "gate_up_proj" in d and "down_proj" in d and d["gate_up_proj"].out_features != 2 * d["down_proj"].in_features:
            raise ValueError(f"{parent}: gate_up_proj / down_proj shards do not line up on rank {tp_rank}")


def fuse_columns(parts: Iterable[PackedGemm]) -> PackedGemm:
    """Concatenate column-parallel linears that share their input (q|k|v, gate|up) along N - what the reference's
    fuse_qkv does for whole tensors (awq/utils/fused_utils.py:67-96), here for the rank's shards."""
    parts = list(parts)
    G = parts[0].group_size
    if any(p.group_size != G or p.in_features != parts[0].in_features for p in parts):
        raise ValueError("fused linears must share in_features and group size")
    bias = None
    if any(p.bias is not None for p in parts):
        bias = torch.cat([p.bias if p.bias is not None else
                          torch.zeros(p.out_features, dtype=torch.float16, device=p.qweight.device) for p in parts])
    return PackedGemm(torch.cat([p.qweight for p in parts], dim=1).contiguous(),
                      torch.cat([p.qzeros for p in parts], dim=1).contiguous(),
                      torch.cat([p.scales for p in parts], dim=1).contiguous(), bias)


def load_stacked_experts(path, prefix: str, E: int, device):
    """The stacked GEMM-layout experts of one MoE block, read from the shards straight into their stacked tensors:
    ((w1 qweight [E, H, 2I/8], scales [E, H/G, 2I], qzeros [E, H/G, 2I/8]), (w2 qweight [E, I, H/8], scales, qzeros)),
    w1 = [gate | up] along N, from `prefix.experts.{e}.{gate,up,down}_proj.*` (Qwen3-MoE / Qwen2-MoE naming).  `path`
    is a checkpoint directory or file, or a CheckpointIndex.  Each shard is opened once and each tensor is copied into
    its place as it is read, so the checkpoint's experts are never held twice.  packing.stack_experts builds the same
    tensors from loaded modules."""
    from safetensors import safe_open

    index = path if isinstance(path, CheckpointIndex) else CheckpointIndex(path)
    kinds = ("qweight", "scales", "qzeros")
    by_file: Dict[str, list] = {}
    for e in range(E):
        for proj in ("gate_proj", "up_proj", "down_proj"):
            for t in kinds:
                name = f"{prefix}.experts.{e}.{proj}.{t}"
                if name not in index.files:
                    raise KeyError(f"{name} is not in the checkpoint")
                by_file.setdefault(index.files[name], []).append((name, e, proj, t))
    w1: Dict[str, torch.Tensor] = {}
    w2: Dict[str, torch.Tensor] = {}
    for file, names in by_file.items():
        with safe_open(file, framework="pt", device="cpu") as f:
            for name, e, proj, t in names:
                x = f.get_tensor(name)
                if proj == "down_proj":
                    if t not in w2:
                        w2[t] = torch.empty((E,) + tuple(x.shape), dtype=x.dtype, device=device)
                    w2[t][e].copy_(x)
                    continue
                n = x.shape[1]
                if t not in w1:
                    w1[t] = torch.empty((E, x.shape[0], 2 * n), dtype=x.dtype, device=device)
                half = slice(0, n) if proj == "gate_proj" else slice(n, 2 * n)
                if w1[t].shape[1:] != (x.shape[0], 2 * n):
                    raise ValueError(f"{name}: shape {tuple(x.shape)} differs from the block's other experts")
                w1[t][e, :, half].copy_(x)
    return tuple(w1[t] for t in kinds), tuple(w2[t] for t in kinds)


def load_shared_expert(path, prefix: str, device):
    """The shared expert of a DeepSeek-MoE block, read next to load_stacked_experts: ((qweight [H, 2 I_s / 8], scales
    [H/G, 2 I_s], qzeros [H/G, 2 I_s / 8]) of [gate | up] along N, (down qweight [I_s, H/8], scales, qzeros)), from
    `prefix.shared_experts.{gate,up,down}_proj.*`.  packing.stack_deepseek_experts builds the same tensors from loaded
    modules."""
    from safetensors import safe_open

    index = path if isinstance(path, CheckpointIndex) else CheckpointIndex(path)
    kinds = ("qweight", "scales", "qzeros")
    got: Dict[str, torch.Tensor] = {}
    by_file: Dict[str, list] = {}
    for proj in ("gate_proj", "up_proj", "down_proj"):
        for t in kinds:
            name = f"{prefix}.shared_experts.{proj}.{t}"
            if name not in index.files:
                raise KeyError(f"{name} is not in the checkpoint")
            by_file.setdefault(index.files[name], []).append(name)
    for file, names in by_file.items():
        with safe_open(file, framework="pt", device="cpu") as f:
            for name in names:
                got[name] = f.get_tensor(name)

    def t(proj, k):
        return got[f"{prefix}.shared_experts.{proj}.{k}"]

    ws1 = tuple(torch.cat((t("gate_proj", k), t("up_proj", k)), dim=1).to(device).contiguous() for k in kinds)
    ws2 = tuple(t("down_proj", k).to(device).contiguous() for k in kinds)
    return ws1, ws2
