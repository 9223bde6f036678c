"""GPU tests of RoPE + KV-cache append for T tokens per sequence (b200awq_rope_kv_seq / b200awq_qk_norm_rope_kv_seq,
ext.rope_kv_cache(seq_len=T), DecodeProgram.rope_kv_cache(seq_len=T)).

Stand-alone: against the reference's RoPE.forward(xq, xk, start_pos, seqlen) and WindowedCache.update_kv (partial
rotary composed as test_gpu_program_partial_rope.py does), the rotated columns within one fp16 ulp (one ulp of the
head's largest value where the products cancel), tails and v bit-exact, every other cache row and entry untouched; Qwen3's q / k norm bit-identical to the one-token op row by row;
T = 1 byte-identical to b200awq_rope_kv.  Programs: Llama- and Qwen3-shaped segments at (B, T) in {(1, 2), (1, 4),
(2, 2)} fused into one launch, every row bit-identical to an M = 1 program on that row at position pos + t into entry
b, the per-op replay, a CUDA graph advancing pos by T, and a step that runs past the end of the cache."""
import pytest
import torch

from test_gpu_program import EPS, _no_abort
from test_gpu_program_qknorm import _norms
from test_gpu_program_rope import _build, _caches, _freqs, _linear, _ulps

pytestmark = pytest.mark.gpu

F16 = torch.float16
THETA = 10000.0
S = 2048
SENT = 7.0


def _dev():
    return torch.device("cuda:0")


def _ref_modules():
    _freqs(8, 8, 1.0)                                       # imports the reference package
    from awq.modules.fused.attn import RoPE
    from awq.modules.fused.cache import WindowedCache

    return RoPE, WindowedCache


def _reference(qkv, rope, cache, H, KV, D, R, B, T, p):
    """The reference's step over tokens [t0, T) that lie inside the cache: RoPE(R).forward on the first R columns of q
    and k with start_pos = p + t0, the tail concatenated back, update_kv.  Returns q [B, T - t0, H, D]."""
    x = qkv.view(B, T, H + 2 * KV, D)
    xq, xk, xv = x[:, :, :H], x[:, :, H:H + KV], x[:, :, H + KV:]
    rq, rk = rope.forward(xq[..., :R].contiguous(), xk[..., :R].contiguous(), p, T)
    q, k = torch.cat((rq, xq[..., R:]), -1), torch.cat((rk, xk[..., R:]), -1)
    cache.update_kv(values_store=xv.contiguous(), keys_store=k.contiguous(), batch_size=B, start_pos=p, seqlen=T)
    return q


def _rotated_close(got, want):
    """Within one fp16 ulp of the reference, or, where the rotation's two products cancel, within one fp16 ulp of the
    head's largest |value| (torch's complex-product loops round such sums differently at large sizes, DESIGN.md 3.5f)."""
    head = want.float().abs().amax(-1, keepdim=True)
    ulp_head = torch.exp2(torch.floor(torch.log2(head.clamp_min(2.0**-14))) - 10)
    near = _ulps(got, want) <= 1
    return bool((near | ((got.float() - want.float()).abs() <= ulp_head)).all())


def _rows_in_range(p, T):
    return [t for t in range(T) if 0 <= p + t < S]


@pytest.mark.parametrize("H,KV,D,R", [(8, 2, 128, 128), (8, 8, 64, 16), (4, 4, 80, 20)])
@pytest.mark.parametrize("T", [1, 2, 3, 4, 8, 37, 512])
def test_seq_matches_reference(H, KV, D, R, T):
    from autoawq_b200 import ext

    RoPE, WindowedCache = _ref_modules()
    rope = RoPE(R, S, _dev(), THETA)
    for B in (1, 2):
        g = torch.Generator(device=_dev()).manual_seed(1000 * T + 10 * D + B)
        qkv = (torch.randn((B, T, (H + 2 * KV) * D), device=_dev(), generator=g) * 3).half()
        for p in sorted({0, 1, 1000, S - T, S - T + 2}):
            if p + T > S + 2 or p < 0:
                continue
            kc, vc = _caches(B + 1, S, KV, D, seed=p + T)     # entry B: a sequence the step does not own
            k0, v0 = kc.clone(), vc.clone()
            q = torch.full((B * T, H, D), SENT, dtype=F16, device=_dev())
            pos = torch.tensor([p], dtype=torch.int32, device=_dev())
            ext.rope_kv_cache(qkv, rope.freqs_cis, pos, kc, vc, H, KV, q_out=q, head_dim=D, seq_len=T)
            torch.cuda.synchronize()
            ts = _rows_in_range(p, T)
            written = torch.zeros((B + 1, S), dtype=torch.bool, device=_dev())
            q = q.view(B, T, H, D)
            if ts:
                t0, n = ts[0], len(ts)
                cache = WindowedCache(B, H, KV, D, S, _dev())
                ref_q = _reference(qkv[:, t0:t0 + n].contiguous().view(B * n, -1), rope, cache, H, KV, D, R, B, n,
                                   p + t0)
                want_k, want_v = cache.k[:, p + t0:p + t0 + n], cache.v[:, p + t0:p + t0 + n]
                got_q, got_k, got_v = q[:, t0:t0 + n], kc[:B, p + t0:p + t0 + n], vc[:B, p + t0:p + t0 + n]
                for got, want, what in ((got_q, ref_q, "q"), (got_k, want_k, "k")):
                    assert _rotated_close(got[..., :R], want[..., :R]), (B, p, what)
                    assert torch.equal(got[..., R:], want[..., R:]), (B, p, what)
                assert torch.equal(got_v, want_v), (B, p)
                written[:B, p + t0:p + t0 + n] = True
            # rows past the end of the cache write nothing, not even q_out
            for t in range(T):
                if t not in ts:
                    assert bool((q[:, t] == SENT).all()), (B, p, t)
            assert torch.equal(kc[~written], k0[~written]) and torch.equal(vc[~written], v0[~written]), (B, p)


@pytest.mark.parametrize("T", [1, 2, 4, 37])
def test_qk_norm_seq_is_the_one_token_op_row_by_row(T):
    from autoawq_b200 import ext

    H, KV, D, B = 8, 2, 128, 2
    freqs = _freqs(D, S, 1e6)
    qn, kn = _norms(D, seed=T)
    g = torch.Generator(device=_dev()).manual_seed(T)
    qkv = (torch.randn((B * T, (H + 2 * KV) * D), device=_dev(), generator=g) * 3).half()
    for p in (0, 1000, S - T, S - T + 2):
        kc, vc = _caches(B + 1, S, KV, D, seed=p)
        rk, rv = kc.clone(), vc.clone()
        q = torch.full((B * T, H, D), SENT, dtype=F16, device=_dev())
        rq = q.clone()
        ext.rope_kv_cache(qkv, freqs, torch.tensor([p], dtype=torch.int32, device=_dev()), kc, vc, H, KV, q_out=q,
                          q_norm=qn, k_norm=kn, seq_len=T)
        for m in range(B * T):
            b, t = divmod(m, T)
            ext.rope_kv_cache(qkv[m:m + 1], freqs, torch.tensor([p + t], dtype=torch.int32, device=_dev()),
                              rk[b:b + 1], rv[b:b + 1], H, KV, q_out=rq[m:m + 1], q_norm=qn, k_norm=kn)
        torch.cuda.synchronize()
        assert torch.equal(q, rq) and torch.equal(kc, rk) and torch.equal(vc, rv), p


def test_t1_is_byte_identical_to_rope_kv():
    from autoawq_b200 import ext
    from autoawq_b200._cabi import lib

    H, KV, D, M = 8, 2, 128, 4
    freqs = _freqs(D, S, THETA)
    qkv = (torch.randn((M, (H + 2 * KV) * D), device=_dev()) * 3).half()
    pos = torch.tensor([77], dtype=torch.int32, device=_dev())
    outs = []
    for seq in (False, True):
        kc, vc = _caches(M, S, KV, D, seed=3)
        q = torch.zeros((M, H, D), dtype=F16, device=_dev())
        r, q2, _ = ext.rope_descriptor(qkv, freqs, pos, kc, vc, H, KV, q)
        s = ext._stream(qkv.device)
        code = (lib.b200awq_rope_kv_seq(q2.data_ptr(), q2.stride(0), r, M, 1, s) if seq else
                lib.b200awq_rope_kv(q2.data_ptr(), q2.stride(0), r, M, s))
        assert code == 0
        torch.cuda.synchronize()
        outs.append((q, kc, vc))
    assert all(torch.equal(a.view(torch.int16), b.view(torch.int16)) for a, b in zip(*outs))


def test_python_checks():
    from autoawq_b200 import ext
    from autoawq_b200._cabi import B200AwqError

    H, KV, D = 4, 2, 64
    freqs = _freqs(D, S, THETA)
    qkv = torch.randn((4, (H + 2 * KV) * D), device=_dev()).half()
    pos = torch.zeros(1, dtype=torch.int32, device=_dev())
    kc, vc = _caches(2, S, KV, D, seed=1)
    ext.rope_kv_cache(qkv, freqs, pos, kc, vc, H, KV, seq_len=2)           # B = 2 entries are enough
    for T in (0, 3, -1):
        with pytest.raises(B200AwqError):
            ext.rope_kv_cache(qkv, freqs, pos, kc, vc, H, KV, seq_len=T)
    with pytest.raises(B200AwqError):                                       # 4 sequences need 4 entries
        ext.rope_kv_cache(qkv, freqs, pos, kc, vc, H, KV, seq_len=1)
    small_k, small_v = _caches(1, S, KV, D, seed=2)
    with pytest.raises(B200AwqError):
        ext.rope_kv_cache(qkv, freqs, pos, small_k, small_v, H, KV, seq_len=2)


# ------------------------------------------------------------------------------------------ decode programs
class Layer:
    """One decoder layer (GEMM-layout AWQ, random weights): Llama-shaped, or Qwen3-shaped with q / k norms."""

    def __init__(self, qwen3, seed, hidden=2048, inter=4096, H=16, KV=4, D=128, G=128):
        self.hidden, self.inter, self.H, self.KV, self.D = hidden, inter, H, KV, D
        self.w = dict(o=_linear(H * D, hidden, G, seed), gu=_linear(hidden, 2 * inter, G, seed + 1),
                      down=_linear(inter, hidden, G, seed + 2), qkv=_linear(hidden, (H + 2 * KV) * D, G, seed + 3))
        g = torch.Generator(device=_dev()).manual_seed(seed + 4)
        self.n1 = (1 + 0.1 * torch.randn(hidden, device=_dev(), generator=g)).half()
        self.n2 = (1 + 0.1 * torch.randn(hidden, device=_dev(), generator=g)).half()
        self.freqs = _freqs(D, S, 1e6 if qwen3 else 500000.0)
        self.norms = dict(zip(("q_norm", "k_norm"), _norms(D, seed + 5))) if qwen3 else {}


def _record(api, L, attn, h_in, pos, kc, vc, T):
    """[o + h, norm2, gate|up, silu, down + h, norm1', qkv', rope_kv_cache(seq_len=T)] against `api`."""
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
    qkv = api.gemm_forward_cuda(xn, *L.w["qkv"], 8)
    q = api.rope_kv_cache(qkv, L.freqs, pos, kc, vc, L.H, L.KV, seq_len=T, **L.norms)
    return dict(o=o, h=h, xn2=xn2, gu=gu, act=act, dn=dn, out=out, xn=xn, qkv=qkv, q=q)


def _inputs(L, M, seed):
    g = torch.Generator(device=_dev()).manual_seed(seed)
    return (torch.randn((M, L.H * L.D), device=_dev(), generator=g).half(),
            torch.randn((M, L.hidden), device=_dev(), generator=g).half())


def _program(L, B, T, pos, kc, vc, seed, no_fuse=False):
    attn, h_in = _inputs(L, B * T, seed)
    return _build(lambda api: _record(api, L, attn, h_in, pos, kc, vc, T), B * T, no_fuse)


def _row_programs(L, B, T, kc, vc, seed):
    """Per row m = b T + t: an M = 1 program on that row alone, at its own position tensor, into entry b."""
    attn, h_in = _inputs(L, B * T, seed)
    rows = []
    for m in range(B * T):
        b = m // T
        pos = torch.zeros(1, dtype=torch.int32, device=_dev())
        prog, bufs = _build(lambda api: _record(api, L, attn[m:m + 1].clone(), h_in[m:m + 1].clone(), pos,
                                                kc[b:b + 1], vc[b:b + 1], 1), 1, False)
        assert prog.fused
        rows.append((pos, prog, bufs))
    return rows


def _check_rows(f, kc, vc, rows, rk, rv, T, what):
    for m, (_, _, r) in enumerate(rows):
        for k in r:
            assert torch.equal(f[k].reshape(len(rows), -1)[m], r[k].reshape(-1)), f"{what}: row {m}, {k}"
    assert torch.equal(kc, rk) and torch.equal(vc, rv), f"{what}: caches"


@pytest.mark.parametrize("qwen3", [False, True], ids=["llama", "qwen3"])
@pytest.mark.parametrize("B,T", [(1, 2), (1, 4), (2, 2)])
def test_program_rows_match_single_token_programs(qwen3, B, T):
    L = Layer(qwen3, seed=10 * B + T)
    pos = torch.zeros(1, dtype=torch.int32, device=_dev())
    kc, vc = _caches(B + 1, S, L.KV, L.D, seed=5)
    rk, rv = kc.clone(), vc.clone()
    prog, f = _program(L, B, T, pos, kc, vc, seed=7)
    assert prog.fused and prog.launches_per_run == 1 and prog.kernel_ops == 4 and prog.tokens == B * T
    rows = _row_programs(L, B, T, rk, rv, seed=7)
    for p in (0, 1000, S - T, S - T + 1):        # the last one runs past the end of the cache
        pos.fill_(p)
        prog.run()
        for m, (rpos, rprog, _) in enumerate(rows):
            rpos.fill_(p + m % T)
            rprog.run()
        torch.cuda.synchronize()
        _no_abort(f"pos {p}")
        _check_rows(f, kc, vc, rows, rk, rv, T, f"pos {p}")


@pytest.mark.parametrize("qwen3", [False, True], ids=["llama", "qwen3"])
def test_per_op_replay_matches(qwen3):
    """Under knob 14 the program replays per op through b200awq_rope_kv_seq: its q and cache rows are the stand-alone
    one-token op row by row on the replay's own qkv, and every buffer is close to the fused run."""
    from autoawq_b200 import ext

    B, T = 2, 2
    L = Layer(qwen3, seed=40)
    pos = torch.zeros(1, dtype=torch.int32, device=_dev())
    kf, vf = _caches(B, S, L.KV, L.D, seed=6)
    kr, vr = kf.clone(), vf.clone()
    fprog, f = _program(L, B, T, pos, kf, vf, seed=8)
    rprog, r = _program(L, B, T, pos, kr, vr, seed=8, no_fuse=True)
    assert fprog.fused and not rprog.fused
    for p in (3, S - T + 1):
        pos.fill_(p)
        k0, v0 = kr.clone(), vr.clone()
        fprog.run()
        rprog.run()
        torch.cuda.synchronize()
        q1 = torch.full_like(r["q"], SENT)
        for m in range(B * T):
            b, t = divmod(m, T)
            ext.rope_kv_cache(r["qkv"][m:m + 1], L.freqs, torch.tensor([p + t], dtype=torch.int32, device=_dev()),
                              k0[b:b + 1], v0[b:b + 1], L.H, L.KV, q_out=q1[m:m + 1], **L.norms)
        torch.cuda.synchronize()
        ok = [t for t in range(T) if p + t < S]
        qr, qw = r["q"].view(B, T, -1)[:, ok], q1.view(B, T, -1)[:, ok]
        assert torch.equal(qr, qw) and torch.equal(kr, k0) and torch.equal(vr, v0), p
        for k in f:
            d = float((f[k].float() - r[k].float()).abs().max())
            assert d <= 0.03 * float(r[k].float().abs().max()) + 0.03, f"pos {p}: {k} differs by {d}"
        assert torch.equal(kf.isfinite(), kr.isfinite())


def test_cuda_graph_advances_by_t():
    B, T = 2, 2
    L = Layer(False, seed=60)
    pos = torch.zeros(1, dtype=torch.int32, device=_dev())
    kc, vc = _caches(B, S, L.KV, L.D, seed=9)
    rk, rv = kc.clone(), vc.clone()
    prog, f = _program(L, B, T, pos, kc, vc, seed=11)
    assert prog.fused
    rows = _row_programs(L, B, T, rk, rv, seed=11)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        prog.run()                                   # warm-up outside the capture (writes rows 0, 1)
    torch.cuda.synchronize()
    for m, (rpos, rprog, _) in enumerate(rows):
        rpos.fill_(m % T)
        rprog.run()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        prog.run()
        pos.add_(T)
    for step in range(4):                            # positions 0, 2, 4, 6 (the first again: same values)
        p = int(pos.item())
        graph.replay()
        for m, (rpos, rprog, _) in enumerate(rows):
            rpos.fill_(p + m % T)
            rprog.run()
        torch.cuda.synchronize()
        _no_abort(f"step {step}")
        _check_rows(f, kc, vc, rows, rk, rv, T, f"step {step}")
    assert int(pos.item()) == 4 * T
