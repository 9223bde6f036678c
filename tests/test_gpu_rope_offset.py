"""GPU tests of RoPE + KV-cache append with a per-sequence rotary offset (b200awq_rope_kv_offset,
ext.rope_kv_cache(rope_offset=), DecodeProgram.rope_kv_cache(rope_offset=)).

Stand-alone: bit-exact against the op without offsets run per sequence at position p + o_b into a scratch cache
(negative, zero and positive offsets, T in {1, 2, 4}, B in {1, 2, 4}, full and partial rotary, with and without Qwen3's
q / k norm, rows whose cache row or rotary position is out of range), against the reference's RoPE.forward at
start_pos p + o_b with WindowedCache.update_kv at p, and against transformers' Qwen2.5-VL apply_multimodal_rotary_pos_emb
with equal 3-D position ids.  Programs: a Qwen2.5-VL-shaped segment (qkv bias) as one launch, all-zero offsets
byte-identical to the program without offsets, Llama- and Qwen3-shaped batched programs row by row against M = 1
programs with each row's own offset, a StableLM segment with an offset fused at M = 1, a CUDA graph replayed while pos
advances and the offsets are rewritten, and the per-op replay."""
import pytest
import torch

from test_gpu_program import EPS, _no_abort
from test_gpu_program_partial_rope import StableLmBlock
from test_gpu_program_partial_rope import _inputs as _stablelm_inputs
from test_gpu_program_qknorm import _norms
from test_gpu_program_rope import _build, _caches, _freqs
from test_gpu_rope_seq import Layer, _inputs, _record, _ref_modules, _rotated_close

pytestmark = pytest.mark.gpu

F16 = torch.float16
S = 2048
SF = S + 64            # frequency rows: a rotary position may lie past the last cache row
SENT = 7.0


def _dev():
    return torch.device("cuda:0")


def _i32(v):
    return torch.tensor(v, dtype=torch.int32, device=_dev())


def _sentinel(*shape):
    return torch.full(shape, SENT, dtype=F16, device=_dev())


class _WithOffset:
    """`api` (ext or a DecodeProgram) whose rope_kv_cache passes rope_offset=off."""

    def __init__(self, api, off):
        self._api, self._off = api, off

    def __getattr__(self, name):
        return getattr(self._api, name)

    def rope_kv_cache(self, *a, **k):
        return self._api.rope_kv_cache(*a, rope_offset=self._off, **k)


# ------------------------------------------------------------------------------------------ stand-alone
GEOMETRIES = [(8, 2, 128, 128, False), (8, 2, 128, 128, True), (8, 8, 64, 16, False), (4, 4, 80, 20, False)]
OFFSETS = [-3, 0, 5, -1000, 70, 1, -2, 0]


@pytest.mark.parametrize("H,KV,D,R,norm", GEOMETRIES, ids=["full", "qk-norm", "partial-64-16", "partial-80-20"])
@pytest.mark.parametrize("T", [1, 2, 4])
@pytest.mark.parametrize("B", [1, 2, 4])
def test_offset_is_the_op_without_offsets_at_the_rotary_position(H, KV, D, R, norm, T, B):
    """Per sequence b: rope_kv_cache(seq_len=T) at position p + o_b into a scratch cache gives q_out bit for bit, and
    its row p + o_b + t is row p + t of entry b.  Caches start sentinel-filled; nothing else changes."""
    from autoawq_b200 import ext

    freqs = _freqs(R, SF, 10000.0)
    norms = dict(zip(("q_norm", "k_norm"), _norms(D, seed=T))) if norm else {}
    g = torch.Generator(device=_dev()).manual_seed(100 * B + 10 * T + D)
    qkv = (torch.randn((B, T, (H + 2 * KV) * D), device=_dev(), generator=g) * 3).half()
    for p in (1, 1000, S - T + 1, S - 40):
        offs = [OFFSETS[(p + b) % len(OFFSETS)] for b in range(B)]
        kc, vc = _sentinel(B + 1, S, KV, D), _sentinel(B + 1, S, KV, D)   # entry B: a sequence the step does not own
        q = _sentinel(B * T, H, D)
        ext.rope_kv_cache(qkv, freqs, _i32([p]), kc, vc, H, KV, q_out=q, head_dim=D, seq_len=T,
                          rope_offset=_i32(offs), **norms)
        written = torch.zeros((B + 1, S), dtype=torch.bool, device=_dev())
        q = q.view(B, T, H, D)
        for b, o in enumerate(offs):
            kx, vx, qx = _sentinel(1, SF, KV, D), _sentinel(1, SF, KV, D), _sentinel(T, H, D)
            ext.rope_kv_cache(qkv[b:b + 1], freqs, _i32([p + o]), kx, vx, H, KV, q_out=qx, head_dim=D, seq_len=T,
                              **norms)
            for t in range(T):
                c, r = p + t, p + t + o
                what = (p, b, t, o)
                if 0 <= c < S and 0 <= r < SF:
                    assert torch.equal(q[b, t], qx[t]), what
                    assert torch.equal(kc[b, c], kx[0, r]) and torch.equal(vc[b, c], vx[0, r]), what
                    written[b, c] = True
                else:                                    # out of range: nothing, not even the q_out row
                    assert bool((q[b, t] == SENT).all()), what
        assert bool((kc[~written] == SENT).all()) and bool((vc[~written] == SENT).all()), p


@pytest.mark.parametrize("H,KV,D,R", [(8, 2, 128, 128), (8, 8, 64, 16)])
@pytest.mark.parametrize("T", [1, 4])
def test_offset_matches_reference(H, KV, D, R, T):
    """The reference's RoPE.forward(xq, xk, start_pos = p + o_b, seqlen = T) and WindowedCache.update_kv at p, for each
    sequence, within the bound the RoPE tests use (test_gpu_rope_seq.py)."""
    from autoawq_b200 import ext

    RoPE, WindowedCache = _ref_modules()
    rope = RoPE(R, S, _dev(), 10000.0)
    B, p = 4, 900
    offs = [-250, 0, 17, 1100]
    g = torch.Generator(device=_dev()).manual_seed(T + D)
    qkv = (torch.randn((B, T, (H + 2 * KV) * D), device=_dev(), generator=g) * 3).half()
    kc, vc = _sentinel(B, S, KV, D), _sentinel(B, S, KV, D)
    q = ext.rope_kv_cache(qkv, rope.freqs_cis, _i32([p]), kc, vc, H, KV, head_dim=D, seq_len=T,
                          rope_offset=_i32(offs)).view(B, T, H, D)
    torch.cuda.synchronize()
    for b, o in enumerate(offs):
        x = qkv[b:b + 1].view(1, T, H + 2 * KV, D)
        xq, xk, xv = x[:, :, :H], x[:, :, H:H + KV], x[:, :, H + KV:]
        rq, rk = rope.forward(xq[..., :R].contiguous(), xk[..., :R].contiguous(), p + o, T)
        wq, wk = torch.cat((rq, xq[..., R:]), -1), torch.cat((rk, xk[..., R:]), -1)
        cache = WindowedCache(1, H, KV, D, S, _dev())
        cache.update_kv(values_store=xv.contiguous(), keys_store=wk.contiguous(), batch_size=1, start_pos=p, seqlen=T)
        got_k, got_v = kc[b:b + 1, p:p + T], vc[b:b + 1, p:p + T]
        for got, want, what in ((q[b:b + 1], wq, "q"), (got_k, cache.k[:, p:p + T], "k")):
            assert _rotated_close(got[..., :R], want[..., :R]), (b, what)
            assert torch.equal(got[..., R:], want[..., R:]), (b, what)
        assert torch.equal(got_v, cache.v[:, p:p + T]), b


def test_offset_matches_transformers_qwen2_5_vl_text_tokens():
    """transformers' Qwen2_5_VLRotaryEmbedding + apply_multimodal_rotary_pos_emb (mrope_section [16, 24, 24]) with the
    three position components all equal to r = p + t + rope_deltas[b], within two fp16 ulps at each head's largest |x|."""
    from autoawq_b200 import ext
    from transformers import Qwen2_5_VLConfig
    from transformers.models.qwen2_5_vl.modeling_qwen2_5_vl import (Qwen2_5_VLRotaryEmbedding,
                                                                    apply_multimodal_rotary_pos_emb)

    H, KV, D, theta, section = 28, 4, 128, 1e6, [16, 24, 24]
    cfg = Qwen2_5_VLConfig(text_config=dict(hidden_size=H * D, num_attention_heads=H, num_key_value_heads=KV,
                                            max_position_embeddings=32768, rope_theta=theta,
                                            rope_scaling={"type": "mrope", "mrope_section": section}))
    rot = Qwen2_5_VLRotaryEmbedding(cfg.text_config, device=_dev())
    freqs = _freqs(D, S + 1024, theta)
    B, T = 2, 2
    g = torch.Generator(device=_dev()).manual_seed(25)
    qkv = (torch.randn((B, T, (H + 2 * KV) * D), device=_dev(), generator=g) * 3).half()
    for p, deltas in ((0, [0, 3]), (1023, [-700, 812]), (S - T, [-5, 1000])):
        kc, vc = _sentinel(B, S, KV, D), _sentinel(B, S, KV, D)
        q = ext.rope_kv_cache(qkv, freqs, _i32([p]), kc, vc, H, KV, seq_len=T, rope_offset=_i32(deltas))
        torch.cuda.synchronize()
        r = torch.tensor([[p + t + d for t in range(T)] for d in deltas], device=_dev())      # [B, T]
        cos, sin = rot(qkv, r[None].expand(3, B, T))
        x = qkv.view(B, T, H + 2 * KV, D).transpose(1, 2)                                       # [B, heads, T, D]
        wq, wk = apply_multimodal_rotary_pos_emb(x[:, :H], x[:, H:H + KV], cos, sin, section)
        want = torch.cat((wq, wk), 1).transpose(1, 2)                                            # [B, T, H + KV, D]
        got = torch.cat((q.view(B, T, H, D), kc[:, p:p + T]), 2)
        diff = (got.float() - want.float()).abs()
        ulp = torch.exp2(torch.floor(torch.log2(want.float().abs().amax(-1, keepdim=True))) - 10)
        assert bool((diff <= 2 * ulp).all()), f"pos {p}: largest difference {float(diff.max())}"
        assert torch.equal(vc[:, p:p + T], qkv.view(B, T, H + 2 * KV, D)[:, :, H + KV:]), p


def test_python_checks():
    from autoawq_b200 import ext
    from autoawq_b200._cabi import B200AwqError

    H, KV, D = 4, 2, 64
    freqs = _freqs(D, S, 10000.0)
    qkv = torch.randn((4, (H + 2 * KV) * D), device=_dev()).half()
    pos = _i32([3])
    kc, vc = _sentinel(2, S, KV, D), _sentinel(2, S, KV, D)
    ext.rope_kv_cache(qkv, freqs, pos, kc, vc, H, KV, seq_len=2, rope_offset=_i32([1, -1]))
    for bad in (_i32([1, 2, 3]), _i32([1]), torch.zeros(2, dtype=torch.int64, device=_dev()), torch.zeros(2,
                dtype=torch.int32), _i32([[1, 2], [3, 4]])[:, 0], [1, 2]):
        with pytest.raises(B200AwqError):
            ext.rope_kv_cache(qkv, freqs, pos, kc, vc, H, KV, seq_len=2, rope_offset=bad)


# ------------------------------------------------------------------------------------------ decode programs
class Qwen2VlLayer(Layer):
    """A Qwen2.5-VL-shaped language-model layer (7 q heads per kv head, qkv bias, rope_theta 1e6), at a reduced width."""

    def __init__(self, seed, hidden=1792, inter=4096, H=14, KV=2, D=128):
        super().__init__(False, seed, hidden, inter, H, KV, D)
        g = torch.Generator(device=_dev()).manual_seed(seed + 9)
        self.bias = (0.1 * torch.randn((H + 2 * KV) * D, device=_dev(), generator=g)).half()
        self.freqs = _freqs(D, S, 1e6)


def _record_qwen2(api, L, attn, h_in, pos, kc, vc, off):
    """_record's Qwen2 block: the qkv linear carries a bias."""
    M = attn.shape[0]
    o = api.gemm_forward_cuda(attn, *L.w["o"], 8)
    h = api.add(o, h_in)
    xn2 = torch.empty((M, L.hidden), dtype=F16, device=_dev())
    api.layernorm_forward_cuda(h, L.n2, xn2, EPS)
    gu = api.gemm_forward_cuda(xn2, *L.w["gu"], 8)
    act = torch.empty((M, L.inter), dtype=F16, device=_dev())
    api.silu_and_mul(act, gu)
    dn = api.gemm_forward_cuda(act, *L.w["down"], 8)
    out = api.add(dn, h)
    xn = torch.empty((M, L.hidden), dtype=F16, device=_dev())
    api.layernorm_forward_cuda(out, L.n1, xn, EPS)
    qkv = api.gemm_forward_cuda(xn, *L.w["qkv"], 8, bias=L.bias)
    q = api.rope_kv_cache(qkv, L.freqs, pos, kc, vc, L.H, L.KV, rope_offset=off)
    return dict(o=o, h=h, xn2=xn2, gu=gu, act=act, dn=dn, out=out, xn=xn, qkv=qkv, q=q)


def _stand_alone(f, L, pos, off, k0, v0, T=1):
    """The stand-alone op with offsets on a program's own qkv (into copies of the caches it started from)."""
    from autoawq_b200 import ext

    q = ext.rope_kv_cache(f["qkv"], L.freqs, pos, k0, v0, L.H, L.KV, seq_len=T, rope_offset=off, **L.norms)
    torch.cuda.synchronize()
    return q


def test_qwen2_5_vl_segment_is_one_launch():
    from autoawq_b200 import ext

    L = Qwen2VlLayer(seed=3)
    pos, off = _i32([1023]), _i32([-389])
    kc, vc = _sentinel(1, S, L.KV, L.D), _sentinel(1, S, L.KV, L.D)
    attn, h_in = _inputs(L, 1, 4)
    prog, f = _build(lambda api: _record_qwen2(api, L, attn, h_in, pos, kc, vc, off), 1, False)
    assert prog.fused and prog.launches_per_run == 1 and prog.kernel_ops == 4
    for p, o in ((1023, -389), (1500, 250), (40, -41)):        # the last one: rotary position -1, nothing written
        pos.fill_(p)
        off.fill_(o)
        k0, v0 = kc.clone(), vc.clone()
        prog.run()
        torch.cuda.synchronize()
        _no_abort(f"pos {p}")
        q0 = _sentinel(1, L.H, L.D)
        ext.rope_kv_cache(f["qkv"], L.freqs, pos, k0, v0, L.H, L.KV, q_out=q0, rope_offset=off)
        torch.cuda.synchronize()
        assert torch.equal(kc, k0) and torch.equal(vc, v0), p
        if p + o >= 0:
            assert torch.equal(f["q"], q0), p


MODELS = {"qwen2.5-vl": lambda seed: Qwen2VlLayer(seed), "llama": lambda seed: Layer(False, seed),
          "qwen3": lambda seed: Layer(True, seed)}


def _record_any(api, L, attn, h_in, pos, kc, vc, T, off):
    if isinstance(L, Qwen2VlLayer):
        assert T == 1
        return _record_qwen2(api, L, attn, h_in, pos, kc, vc, off)
    return _record(_WithOffset(api, off), L, attn, h_in, pos, kc, vc, T)


@pytest.mark.parametrize("model,B,T", [("qwen2.5-vl", 1, 1), ("qwen2.5-vl", 2, 1), ("llama", 1, 1), ("llama", 2, 2),
                                       ("qwen3", 1, 1), ("qwen3", 2, 2)])
def test_zero_offsets_are_the_program_without_offsets(model, B, T):
    L = MODELS[model](seed=20 + B + T)
    M = B * T
    attn, h_in = _inputs(L, M, 5)
    pos = _i32([1000])
    outs = []
    for off in (None, _i32([0] * B)):
        kc, vc = _sentinel(B, S, L.KV, L.D), _sentinel(B, S, L.KV, L.D)
        prog, f = _build(lambda api: _record_any(api, L, attn, h_in, pos, kc, vc, T, off), M, False)
        assert prog.fused and prog.launches_per_run == 1
        prog.run()
        torch.cuda.synchronize()
        _no_abort(model)
        outs.append(dict(f, k=kc, v=vc))
    for k in outs[0]:
        assert torch.equal(outs[0][k].view(torch.int16), outs[1][k].view(torch.int16)), k


def _row_programs(L, B, T, kc, vc, attn, h_in):
    """Per row m = b T + t: an M = 1 program on that row alone, with its own position and offset tensors, into entry
    b."""
    rows = []
    for m in range(B * T):
        b = m // T
        pos, off = _i32([0]), _i32([0])
        prog, bufs = _build(lambda api: _record_any(api, L, attn[m:m + 1].clone(), h_in[m:m + 1].clone(), pos,
                                                    kc[b:b + 1], vc[b:b + 1], 1, off), 1, False)
        assert prog.fused
        rows.append((pos, off, prog, bufs))
    return rows


def _run_rows(rows, p, offs, T):
    for m, (rpos, roff, rprog, _) in enumerate(rows):
        rpos.fill_(p + m % T)
        roff.fill_(offs[m // T])
        rprog.run()


def _check_rows(f, kc, vc, rows, rk, rv, what):
    for m, (_, _, _, r) in enumerate(rows):
        for k in r:
            assert torch.equal(f[k].reshape(len(rows), -1)[m], r[k].reshape(-1)), f"{what}: row {m}, {k}"
    assert torch.equal(kc, rk) and torch.equal(vc, rv), f"{what}: caches"


@pytest.mark.parametrize("qwen3", [False, True], ids=["llama", "qwen3"])
@pytest.mark.parametrize("B,T", [(2, 1), (4, 1), (1, 4), (2, 2)])
def test_batched_rows_match_single_row_programs(qwen3, B, T):
    L = Layer(qwen3, seed=30 + 10 * B + T)
    attn, h_in = _inputs(L, B * T, 7)
    pos, off = _i32([0]), _i32([0] * B)
    kc, vc = _sentinel(B + 1, S, L.KV, L.D), _sentinel(B + 1, S, L.KV, L.D)
    rk, rv = kc.clone(), vc.clone()
    prog, f = _build(lambda api: _record_any(api, L, attn, h_in, pos, kc, vc, T, off), B * T, False)
    assert prog.fused and prog.launches_per_run == 1 and prog.kernel_ops == 4 and prog.tokens == B * T
    rows = _row_programs(L, B, T, rk, rv, attn, h_in)
    for p, offs in ((3, [0, -3, 250, -1][:B]), (1000, [-17, 40, 0, 3][:B]), (S - T + 1, [5, -250, 1, 0][:B])):
        pos.fill_(p)
        off.copy_(_i32(offs))
        prog.run()
        _run_rows(rows, p, offs, T)
        torch.cuda.synchronize()
        _no_abort(f"pos {p}")
        _check_rows(f, kc, vc, rows, rk, rv, f"pos {p}")


@pytest.mark.parametrize("model", ["stablelm-3b-4e1t"])
def test_stablelm_segment_with_offset_is_fused(model):
    from autoawq_b200 import ext

    blk = StableLmBlock(model, seed=11)
    attn, x = _stablelm_inputs(blk, 1, 3)
    pos, off = _i32([5]), _i32([20])
    prog, f = _build(lambda api: blk.record(_WithOffset(api, off), pos, attn, x), 1, False)
    assert prog.fused and prog.kernel_ops == 4 and prog.launches_per_run == 1
    prog.run()
    torch.cuda.synchronize()
    _no_abort(model)
    k0, v0 = _caches(1, blk.S, blk.KV, blk.D, 5)                 # the caches record() started from
    rq = ext.rope_kv_cache(f["qkv"], blk.freqs, pos, k0, v0, blk.H, blk.KV, head_dim=blk.D, rope_offset=off)
    torch.cuda.synchronize()
    assert torch.equal(f["q"], rq) and torch.equal(f["k"], k0) and torch.equal(f["v"], v0)


def test_cuda_graph_follows_pos_and_rewritten_offsets():
    B, T = 2, 2
    L = Layer(False, seed=60)
    attn, h_in = _inputs(L, B * T, 11)
    pos, off = _i32([0]), _i32([0, 0])
    kc, vc = _sentinel(B, S, L.KV, L.D), _sentinel(B, S, L.KV, L.D)
    rk, rv = kc.clone(), vc.clone()
    prog, f = _build(lambda api: _record_any(api, L, attn, h_in, pos, kc, vc, T, off), B * T, False)
    assert prog.fused
    rows = _row_programs(L, B, T, rk, rv, attn, h_in)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        prog.run()                                   # warm-up outside the capture (rows 0, 1 at offset 0)
    torch.cuda.synchronize()
    _run_rows(rows, 0, [0, 0], T)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        prog.run()
        pos.add_(T)
    for step, offs in enumerate(([0, 0], [-2, 9], [31, -1], [0, 100])):
        p = int(pos.item())
        off.copy_(_i32(offs))                        # rewritten in place between replays
        graph.replay()
        _run_rows(rows, p, offs, T)
        torch.cuda.synchronize()
        _no_abort(f"step {step}")
        _check_rows(f, kc, vc, rows, rk, rv, f"step {step}")
    assert int(pos.item()) == 4 * T


@pytest.mark.parametrize("model,B,T", [("qwen2.5-vl", 1, 1), ("llama", 2, 2), ("qwen3", 2, 2)])
def test_per_op_replay_gives_the_stand_alone_rows(model, B, T):
    """Under knob 14 the program replays per op through b200awq_rope_kv_offset: its q and cache rows are the stand-alone
    op on the replay's own qkv."""
    L = MODELS[model](seed=40)
    attn, h_in = _inputs(L, B * T, 8)
    pos, off = _i32([600]), _i32([-31, 77][:B])
    kc, vc = _sentinel(B, S, L.KV, L.D), _sentinel(B, S, L.KV, L.D)
    prog, r = _build(lambda api: _record_any(api, L, attn, h_in, pos, kc, vc, T, off), B * T, True)
    assert not prog.fused
    k0, v0 = kc.clone(), vc.clone()
    prog.run()
    torch.cuda.synchronize()
    q1 = _stand_alone(r, L, pos, off, k0, v0, T)
    assert torch.equal(r["q"], q1) and torch.equal(kc, k0) and torch.equal(vc, v0)
