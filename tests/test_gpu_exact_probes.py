"""Exact-arithmetic probes of every linear kernel route (oracle/exact_probe.py; DESIGN.md section 4).

The data are integers times powers of two, sized so that the true output is an fp16 value and every partial sum is
exact in fp32: any summation order returns the same bits, and every check below is equality of the fp16 VALUES over
the whole output (values, not bits: split-K sums start from +0, so a -0 may come back as +0).  A kernel that drops,
duplicates or misplaces one k-row, one column set or one token row at a tile, warp, K-split, ring or unit boundary
changes an output by at least one unit and fails; the failure message lists the first wrong (row, column) pairs and
the difference in units, which locates the boundary.

Activation rows are sparse (the output must stay within 2048 units), and the supports of consecutive rows partition
0..K-1: calls with fewer rows than `cover_rows` are repeated over successive row chunks until the union of their
supports is every k (100 % coverage for M <= 8; the first and the last chunk above that).
"""
import functools

import numpy as np
import pytest
import torch

from oracle import awq_oracle as O
from oracle import exact_probe as E

pytestmark = pytest.mark.gpu

MODEL_SHAPES = [
    ("8b.qkv", 4096, 6144), ("8b.o", 4096, 4096), ("8b.gate_up", 4096, 28672), ("8b.down", 14336, 4096),
    ("70b8.qkv", 8192, 1280), ("70b8.o", 1024, 8192), ("70b8.gate_up", 8192, 7168), ("70b8.down", 3584, 8192),
]
# N % 256 != 0 (1936, 96, 40, 384, 640), K % 128 != 0 (384, 1152, 576), G in {32, 64, 128, K}, K / G = 3 and 9 (padded
# zeros width of the GEMV layouts)
EDGE_SHAPES = [(1024, 1936, 128), (512, 96, 128), (256, 40, -1), (384, 256, 128), (1152, 384, 128), (1152, 384, 64),
               (512, 256, 32), (2048, 640, -1), (576, 128, 64)]
# 1-4: each token variant of the persistent GEMV; 5-128: every token tile of the small-M kernel; 129, 160: the wgmma
# GEMM with split-K; 256-300: without
MS = [1, 2, 3, 4, 5, 8, 9, 16, 17, 33, 64, 65, 128, 129, 160, 256, 257, 300]
ROWS = 300


def _dev():
    return torch.device("cuda:0")


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(_dev())


@pytest.fixture(scope="module")
def ext():
    import awq_ext  # noqa: F401
    from autoawq_b200 import ext as e

    return e


@functools.lru_cache(maxsize=6)
def _case(K, N, G, rows=ROWS):
    """One probe per (K, N, G), reused over M by slicing rows; with a bias (y_exact includes it)."""
    n = E.make_exact_case(K, N, G, 1, seed=K % 97 + N % 89, bias=True, layouts=(), reference=False)["cover_rows"]
    return E.make_exact_case(K, N, G, max(rows, n), seed=K % 97 + N % 89, bias=True)


class Probe:
    """A case on the device: weights in the three layouts, all activation rows, and the exact outputs as fp16."""

    def __init__(self, c, layouts=("gemm", "gemv", "fast")):
        self.c, self.K, self.G, self.unit = c, c["x"].shape[1], c["group_size"], c["unit"]
        self.x = _t(c["x"])
        self.bias = _t(c["bias"])
        self.y_bias = _t(c["y_exact"].astype(np.float16))
        self.y_plain = _t((c["y_exact"] - c["bias"].astype(np.float64)).astype(np.float16))
        self.w = {}
        if "gemm" in layouts:
            self.w["gemm"] = (_t(c["qweight"]), _t(c["scales"]), _t(c["qzeros"]))
        if "gemv" in layouts:
            vw, vz, vs = c["gemv"]
            self.w["gemv"] = (_t(vw), _t(vs), _t(vz))
        if "fast" in layouts:
            fw, fs, fz = c["fast"]
            self.w["fast"] = (_t(fw), _t(fs), _t(fz))

    def chunks(self, M):
        """Row ranges of M rows: all of a cover for M <= 8, else its first and last chunk; one range when M rows
        already cover every k."""
        cover, total = self.c["cover_rows"], self.x.shape[0]
        if M >= cover:
            return [(7 * M) % (total - M + 1)]
        starts = list(range(0, cover, M))
        starts = [min(s, total - M) for s in starts]
        return starts if M <= 8 else [starts[0], starts[-1]]

    def want(self, r0, M, bias):
        return (self.y_bias if bias else self.y_plain)[r0:r0 + M]

    def check(self, y, r0, M, bias, what):
        want = self.want(r0, M, bias)
        assert tuple(y.shape) == tuple(want.shape) and y.dtype == torch.float16, what
        if bool((y == want).all()):
            return
        raise AssertionError(f"{what}, rows {r0}..{r0 + M - 1}: "
                             + E.mismatch_report(y.cpu().numpy(), want.cpu().numpy(), self.unit))

    def forward(self, ext, layout, r0, M, bias, x=None):
        xr = self.x[r0:r0 + M] if x is None else x
        return ext.linear_forward(layout, xr, *self.w[layout], self.G, self.bias if bias else None)


def _workspace_is_zero(ext):
    torch.cuda.synchronize()
    for ws in ext._WS.values():
        assert int(ws.view(torch.int32).ne(0).sum()) == 0, "split-K scratch not restored to zero"


def _all_layouts(ext, p, Ms, tag, layouts=("gemm", "gemv", "fast")):
    for M in Ms:
        for i, r0 in enumerate(p.chunks(M)):
            for j, layout in enumerate(layouts):
                bias = (i + j) % 2 == 0                # with and without, on every layout over the chunks / the Ms
                what = f"{tag} {layout} layout M={M} bias={bias}"
                p.check(p.forward(ext, layout, r0, M, bias), r0, M, bias, what)
                if i == 0:
                    p.check(p.forward(ext, layout, r0, M, not bias), r0, M, not bias, what + " (other bias setting)")
    _workspace_is_zero(ext)


def _awq_names(p, tag):
    """The same probes through the drop-in operator names."""
    import awq_ext
    import awq_v2_ext

    K, G, N = p.K, p.G, p.y_plain.shape[1]
    for M in (1, 8, 40):
        r0 = p.chunks(M)[0]
        x = p.x[r0:r0 + M]
        p.check(awq_ext.gemm_forward_cuda(x, *p.w["gemm"], 8), r0, M, False, f"{tag} awq_ext.gemm_forward_cuda M={M}")
        if "gemv" in p.w:
            f = awq_ext.gemmv2_forward_cuda if M > 8 else awq_ext.gemv_forward_cuda
            y = f(x, *p.w["gemv"], G, 8) if M > 8 else f(x, *p.w["gemv"], G)
            p.check(y, r0, M, False, f"{tag} awq_ext gemv-layout entry M={M}")
        if "fast" in p.w and G in (32, 64, 128):
            if M > 8:
                y = awq_v2_ext.gemm_forward_cuda_prefill(x.unsqueeze(0), *p.w["fast"])[0]
            else:
                y = awq_v2_ext.gemv_forward_cuda_decode(x.unsqueeze(1), *p.w["fast"], M, N, K, G)[:, 0]
            p.check(y, r0, M, False, f"{tag} awq_v2_ext entry M={M}")


def _strided_and_repeated(ext, p, tag, layouts):
    for M in (2, 40, 200):
        r0 = p.chunks(M)[0]
        wide = torch.zeros((M, 2 * p.K), dtype=torch.float16, device=_dev())
        wide[:, p.K:] = 3.0                                     # a kernel that ignores the row pitch reads these
        xs = wide[:, :p.K]
        xs.copy_(p.x[r0:r0 + M])
        assert xs.stride(0) == 2 * p.K
        for layout in layouts:
            for rep in range(2):                                # twice in a row: the scratch was restored
                p.check(p.forward(ext, layout, r0, M, True, x=xs), r0, M, True,
                        f"{tag} {layout} layout M={M} row pitch 2K, call {rep}")
    _workspace_is_zero(ext)


def _dequant_bit_exact(p, tag):
    import awq_ext

    c = p.c
    w = O.dequantize_gemm(c["qweight"], c["qzeros"], c["scales"], p.G)
    wd = awq_ext.dequantize_weights_cuda(*p.w["gemm"], 0, 0, 0, False).cpu().numpy()
    assert np.array_equal(wd.view(np.uint16), w.view(np.uint16)), f"{tag}: dequant not bit-exact"
    assert np.array_equal(wd.astype(np.float64), c["w_units"] * c["unit"])


@pytest.mark.parametrize("name,K,N", MODEL_SHAPES)
def test_linear_exact_at_model_shapes(ext, name, K, N):
    p = Probe(_case(K, N, 128))
    _all_layouts(ext, p, MS, name)
    _awq_names(p, name)
    _strided_and_repeated(ext, p, name, ("gemm", "gemv", "fast"))
    if K * N <= 4096 * 6144:
        _dequant_bit_exact(p, name)


@pytest.mark.parametrize("K,N,G", EDGE_SHAPES)
def test_linear_exact_at_envelope_edges(ext, K, N, G):
    # the GEMV / GEMVFast layouts are exercised where N is a multiple of 32, as their other tests do
    layouts = ("gemm", "gemv", "fast") if N % 32 == 0 else ("gemm",)
    p = Probe(E.make_exact_case(K, N, G, ROWS, seed=K + N, bias=True, zero_col_frac=0.05, layouts=layouts), layouts)
    tag = f"K={K} N={N} G={p.G}"
    _all_layouts(ext, p, MS, tag, layouts)
    if len(layouts) == 3:
        _awq_names(p, tag)
    _strided_and_repeated(ext, p, tag, layouts)
    _dequant_bit_exact(p, tag)


ROUTES = [
    # knob, value, Ms, what the knob selects
    (5, 1, (1, 2, 3, 4, 8), "register-staged GEMV"),
    (19, 1, (9, 16, 33, 64, 128), "register-staged wgmma kernel below 129 tokens"),
    (2, 0, (1, 3, 4, 8), "small-M kernel down to M = 1"),
    (21, 1, (5, 9, 16, 17, 64, 128), "small-M kernel, work cut 1"),
    (21, 2, (5, 9, 16, 17, 64, 128), "small-M kernel, work cut 2"),
    (18, 1, (1,), "fp32-RED split-K at M = 1"),
    (4, 1, (1, 4, 16, 300), "programmatic dependent launch"),
]


@pytest.mark.parametrize("knob,value,Ms,what", ROUTES)
@pytest.mark.parametrize("K,N,G", [(4096, 4096, 128), (14336, 4096, 128), (2048, 768, 128), (1152, 384, 64)])
def test_linear_exact_on_alternative_routes(ext, knob, value, Ms, what, K, N, G):
    p = Probe(_case(K, N, G), ("gemm",))
    prev = ext.get_knob(knob)
    ext.set_knob(knob, value)
    try:
        for M in Ms:
            for r0 in p.chunks(M):
                tag = f"knob {knob} = {value} ({what}) K={K} N={N} M={M}"
                y1 = p.forward(ext, "gemm", r0, M, True)
                y2 = p.forward(ext, "gemm", r0, M, False)       # back to back: the second launch overlaps the first
                p.check(y1, r0, M, True, tag)
                p.check(y2, r0, M, False, tag + " second call")
        _workspace_is_zero(ext)
    finally:
        ext.set_knob(knob, prev)


def test_prefill_exact_on_all_rows(ext):
    """One 4096-token call at 4096 x 4096, every row and column, in the three layouts."""
    K = N = 4096
    p = Probe(E.make_exact_case(K, N, 128, 4096, seed=5, bias=True))
    for layout in ("gemm", "gemv", "fast"):
        p.check(p.forward(ext, layout, 0, 4096, True), 0, 4096, True, f"prefill 4096 x 4096 x 4096, {layout} layout")
    _workspace_is_zero(ext)


# ------------------------------------------------------------------------------------------------ MoE operators
class Experts:
    """E exact experts that share one set of activation rows: y for any (row, expert) pair is exact."""

    def __init__(self, E_, K, N, G, rows, seed):
        cs = [E.make_exact_case(K, N, G, rows if e == 0 else 1, seed=seed + e, layouts=("gemm",), reference=False)
              for e in range(E_)]
        self.unit, self.G = cs[0]["unit"], cs[0]["group_size"]
        self.x_units, self.x = cs[0]["x_units"], cs[0]["x"]
        self.w_units = [c["w_units"] for c in cs]
        assert int(np.abs(self.x_units).astype(np.int64).sum(axis=1).max()) * 60 < E.PARTIAL_LIMIT
        self.dev = tuple(_t(np.stack([c[k] for c in cs])) for k in ("qweight", "scales", "qzeros"))

    def y_units(self, row, e):
        y = E.contract_units(self.x_units[row:row + 1], self.w_units[e])[0]
        assert np.abs(y).max() <= E.FP16_EXACT_INT
        return y


def _routing(T, topk, E_, rng):
    ids = np.stack([rng.permutation(E_)[:topk] for _ in range(T)]).astype(np.int32)
    tw = (2.0 ** rng.integers(-3, 1, size=(T, topk))).astype(np.float32)       # 1/8 .. 1: products stay fp16 values
    s, e, n = O.moe_align_block_size(ids, 16, E_)
    return ids, tw, _t(s), _t(np.where(e < 0, 0, e).astype(np.int32)), _t(np.array([n], dtype=np.int32))


def _grouped_exact(ext, ex, T, topk, E_, per_slot, mul, rng, tag):
    ids, tw, s_ids, e_ids, npost = _routing(T, topk, E_, rng)
    K = ex.x.shape[1]
    if per_slot:
        x = _t(ex.x[:T * topk]).view(T, topk, K)
    else:
        x = _t(ex.x[:T]).view(T, 1, K)
    y = ext.grouped_gemm_forward(x, *ex.dev, _t(tw), s_ids, e_ids, npost, mul, 8)
    want = np.stack([np.stack([ex.y_units(t * topk + k if per_slot else t, ids[t, k]) * ex.unit
                               * (float(tw[t, k]) if mul else 1.0) for k in range(topk)]) for t in range(T)])
    assert np.array_equal(want.astype(np.float16).astype(np.float64), want)
    assert tuple(y.shape) == want.shape, tag                   # one row per real slot, no padding rows
    got = y.cpu().numpy().astype(np.float64)
    N = want.shape[-1]
    if not np.array_equal(got, want):
        raise AssertionError(f"{tag}: (row = token * topk + slot) "
                             + E.mismatch_report(got.reshape(-1, N), want.reshape(-1, N), ex.unit / 8))


@pytest.mark.parametrize("E_,topk,K,N,G,knob12,kernel", [
    (8, 2, 1024, 512, 128, 0, "ring"), (4, 2, 512, 256, 64, 0, "ring"),
    (6, 3, 1536, 96, 128, 0, "register-staged (N % 256 != 0)"), (8, 2, 1024, 512, 128, 2, "register-staged (knob 12 = 2)"),
])
def test_grouped_gemm_exact(ext, E_, topk, K, N, G, knob12, kernel):
    ex = Experts(E_, K, N, G, 300 * topk, seed=40)
    rng = np.random.default_rng(E_ + K)
    ext.set_knob(12, knob12)
    try:
        for T in (1, 2, 3, 5, 37, 300):
            for per_slot in (False, True):
                for mul in (False, True):
                    _grouped_exact(ext, ex, T, topk, E_, per_slot, mul, rng,
                                   f"grouped GEMM, {kernel}, T={T} x per slot={per_slot} mul_weights={mul}")
    finally:
        ext.set_knob(12, 0)
    _workspace_is_zero(ext)


@pytest.mark.parametrize("K,N", [(4096, 28672), (14336, 4096)])
def test_grouped_gemm_exact_at_mixtral_shapes(ext, K, N):
    ex = Experts(8, K, N, 128, 10, seed=60)
    rng = np.random.default_rng(K)
    per_slot = K == 14336                                       # the down op reads one activation row per slot
    for T in (1, 5):
        _grouped_exact(ext, ex, T, 2, 8, per_slot, per_slot, rng, f"Mixtral expert {K} x {N}, T={T}")
    _workspace_is_zero(ext)


# ---------------------------------------------------------------------------------------------- stream programs
FAMILIES = {
    "llama-3-8b": [(4096, 6144), (4096, 4096), (4096, 28672), (14336, 4096)],
    "qwen3-8b": [(4096, 6144), (4096, 4096), (4096, 24576), (12288, 4096)],
    "llama-3-70b / 8 ranks": [(8192, 1280), (1024, 8192), (8192, 7168), (3584, 8192)],
}


def _fits_fused(M, Ks):
    """The batched kernel keeps M activation rows of the deepest op in shared memory: at 8 tokens a K of 12288 or
    more does not fit next to the weight ring (DESIGN.md 3.5c), and the program replays per op - still exact."""
    return M < 8 or max(Ks) < 12288


def _no_abort(tag):
    from autoawq_b200.program import DecodeProgram

    rec = DecodeProgram.abort_record()
    assert rec[3] == 0, f"{tag}: program kernel gave up waiting: code={rec[0]} op={rec[1]} cta={rec[2]}"


def _set_knobs(ext, knobs):
    prev = {k: ext.get_knob(k) for k in knobs}
    for k, v in knobs.items():
        ext.set_knob(k, v)
    return prev


@pytest.mark.parametrize("knobs,fused", [({}, True), ({9: 12}, True), ({8: 16}, True), ({14: 1}, False)],
                         ids=["default", "knob9=12", "knob8=16", "knob14=1-replay"])
@pytest.mark.parametrize("M", [1, 2, 3, 4, 8])
@pytest.mark.parametrize("family", list(FAMILIES))
def test_program_of_independent_linears_exact(ext, family, M, knobs, fused):
    """Eight linears (a block's four, twice) on external exact rows in one program: the weight ring crosses seven op
    boundaries.  Every token row of every op against the exact reference, over as many runs as it takes the rows'
    supports to cover every k of the deepest op."""
    from autoawq_b200.program import DecodeProgram

    probes = [Probe(_case(K, N, 128), ("gemm",)) for K, N in FAMILIES[family]]
    prev = _set_knobs(ext, knobs)
    try:
        prog = DecodeProgram(max_tokens=M)
        xs, ys = [], []
        for i in range(8):
            p = probes[i % 4]
            xb = torch.zeros((M, p.K), dtype=torch.float16, device=_dev())
            xs.append(xb)
            ys.append(prog.gemm_forward_cuda(xb, *p.w["gemm"], 8, bias=p.bias if i % 2 else None))
        prog.build()
        fused = fused and _fits_fused(M, [K for K, _ in FAMILIES[family]])
        assert prog.fused == fused, f"{family} M={M}: fused={prog.fused}"
        assert prog.kernel_ops == (8 if fused else 0)
        runs = max(-(-p.c["cover_rows"] // M) for p in probes)
        for run in range(runs):
            r0s = []
            for i in range(8):
                p = probes[i % 4]
                # the second copy of an op walks the rows from the other end
                r0 = (run * M + (i // 4) * 17) % (p.x.shape[0] - M + 1)
                r0s.append(r0)
                xs[i].copy_(p.x[r0:r0 + M])
            prog.run()
            for i in range(8):
                probes[i % 4].check(ys[i].view(M, -1), r0s[i], M, bool(i % 2),
                                    f"{family} program M={M} knobs={knobs} run {run} op {i}")
        if fused:
            _no_abort(f"{family} M={M}")
        prog.close()
    finally:
        _set_knobs(ext, prev)


@pytest.mark.parametrize("M", [1, 2, 4, 8])
@pytest.mark.parametrize("replay", [0, 1])
def test_program_silu_and_residual_exact(ext, M, replay):
    """A linear with an external residual add, then gate|up with SiLU * mul folded in (stream format mode 1).  g and u
    are exactly known integers, so `gate_up` is compared exactly and `act` with fp64 silu(g) * u under 2 fp16 ulps,
    with no K-proportional term; sums of integers are exact, so both the add's output and the producer's raw y are."""
    from autoawq_b200.program import DecodeProgram

    H, I = 4096, 14336
    pg, po, pd = (Probe(_case(K, N, 128), ("gemm",)) for K, N in ((H, 2 * I), (H, H), (I, H)))
    prev = _set_knobs(ext, {14: replay})
    try:
        prog = DecodeProgram(max_tokens=M)
        xg = torch.zeros((M, H), dtype=torch.float16, device=_dev())
        xo = torch.zeros((M, H), dtype=torch.float16, device=_dev())
        res = torch.zeros((M, H), dtype=torch.float16, device=_dev())
        y = prog.gemm_forward_cuda(xo, *po.w["gemm"], 8)
        h = prog.add(res, y)
        gu = prog.gemm_forward_cuda(xg, *pg.w["gemm"], 8)
        act = torch.empty((M, I), dtype=torch.float16, device=_dev())
        prog.silu_and_mul(act, gu)
        # SiLU * mul folds into gate|up only with the linear that consumes `act` behind it; `act` is not exact, so
        # this linear's output stays with the tolerance tests (tests/test_gpu_program.py)
        prog.gemm_forward_cuda(act, *pd.w["gemm"], 8)
        prog.build()
        fused = not replay and _fits_fused(M, [I])
        assert prog.fused == fused and prog.kernel_ops == (3 if fused else 0)
        for run in range(-(-pg.c["cover_rows"] // M)):
            r0 = run * M
            xg.copy_(pg.x[r0:r0 + M])
            xo.copy_(po.x[r0:r0 + M])
            # the residual: the probe's bias, rotated differently per token row (|y + residual| stays within 2048 units)
            shifts = [r0 + m + 1 for m in range(M)]
            res.copy_(torch.stack([torch.roll(po.bias, s) for s in shifts]))
            prog.run()
            tag = f"program M={M} replay={replay} run {run}"
            pg.check(gu.view(M, -1), r0, M, False, tag + " gate|up")
            po.check(y.view(M, -1), r0, M, False, tag + " producer of the add")
            want_h = po.y_plain[r0:r0 + M].double() + res.double()
            assert bool((h.view(M, -1).double() == want_h).all()), tag + ": residual add is not exact: " + \
                E.mismatch_report(h.view(M, -1).cpu().numpy(), want_h.cpu().numpy(), po.unit)
            g64 = pg.y_plain[r0:r0 + M, :I].double()
            want_act = g64 / (1 + torch.exp(-g64)) * pg.y_plain[r0:r0 + M, I:].double()
            ulp = torch.maximum(2.0 ** (torch.floor(torch.log2(want_act.abs().clamp_min(2.0**-14))) - 10),
                                torch.tensor(2.0**-24, dtype=torch.float64, device=_dev()))
            err = (act.double() - want_act).abs()
            assert bool((err <= 2 * ulp).all()), f"{tag} act: {int((err > 2 * ulp).sum())} elements beyond 2 ulps, " \
                                                 f"max {float((err / ulp).max()):.2f} ulps"
        if fused:
            _no_abort(f"silu + residual M={M}")
        prog.close()
    finally:
        _set_knobs(ext, prev)
