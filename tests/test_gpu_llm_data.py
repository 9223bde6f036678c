"""The W4A16 kernels against fp64 on LLM-shaped data (oracle/llm_data.make_llm_case): massive activation channels,
zero-point-heavy codes with all-zero columns and groups, tiny / subnormal / unit scales, outputs at the fp16 range
limit, split-K partials beyond fp16 that cancel, and non-finite or poisoned activations.

Every check holds a route to oracle/llm_data.forward_tolerance of the family of the kernel that ran.  Route-to-family
map (cabi.cu:127-190, restated in oracle/llm_data.*_route_family):

  GEMM layout     M <= 4 (M <= 8 where the small-M wgmma kernel does not apply, or with knob 19 = 1)
                    gemv_v3 (default) / register-staged GEMV (knob 5 = 1) .................... offset-fold
                  otherwise, and every M with knob 2 = 0: the small-M kernel (M <= 128) or the
                    wgmma GEMM, any work cut (knob 21), any split-K epilogue ..................... exact-dequant
  GEMV layout     M <= 2: warp-per-row kernel ................................................ code-fold
                  M > 2: wgmma GEMM with the GEMV-layout loader ................................ exact-dequant
  GEMVFast layout M <= 2: warp-per-row kernel ................................................ code-fold
                  M > 2: wgmma GEMM with the GEMVFast loader (fp16(q s + sz) per weight) ...... fast-dequant
  grouped GEMM    T * topk >= 20 E: moe_tc_kernel ............................................ exact-dequant
                  otherwise gemv_v3_moe, or moe_grouped_kernel (knob 12 = 2, or N % 256 != 0) ... offset-fold
  decode program  stream / batched kernels ................................................... offset-fold

Columns are checked on a sample (every 61st plus the tile edges) that always holds every designated column.  The
largest error / bound ratio per family and route is printed at the end of the module (pytest -s)."""
import numpy as np
import pytest
import torch

from oracle import awq_oracle as O
from oracle import llm_data as L

pytestmark = pytest.mark.gpu

G = 128
ROWS = 300
SHAPES = [
    ("8b.qkv", 4096, 6144), ("8b.o", 4096, 4096), ("8b.gate_up", 4096, 28672), ("8b.down", 14336, 4096),
    ("70b8.qkv", 8192, 1280), ("70b8.o", 1024, 8192), ("70b8.gate_up", 8192, 7168), ("70b8.down", 3584, 8192),
]
MS = [1, 2, 3, 4, 5, 8, 9, 16, 64, 128, 129, 300]
ROUTES = [
    # knob, value, Ms, what the knob selects (test_gpu_exact_probes.py)
    ({5: 1}, (1, 2, 3, 4, 8), "register-staged GEMV"),
    ({2: 0}, (1, 3, 4, 8), "small-M kernel down to M = 1"),
    ({19: 1}, (5, 8, 9, 16, 64, 128), "register-staged wgmma kernel below 129 tokens"),
    ({21: 1}, (5, 9, 16, 17, 64, 128), "small-M kernel, work cut 1"),
    ({21: 2}, (5, 9, 16, 17, 64, 128), "small-M kernel, work cut 2"),
    ({18: 1}, (1,), "fp32-RED split-K at M = 1"),
    ({4: 1}, (1, 4, 16, 300), "programmatic dependent launch"),
]
RATIOS: dict = {}


def _dev():
    return torch.device("cuda:0")


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(_dev())


@pytest.fixture(scope="module")
def ext():
    import awq_ext  # noqa: F401
    from autoawq_b200 import ext as e

    return e


class Linear:
    """One LLM-shaped case on the device in the three layouts, with its fp64 truth on a column sample."""

    def __init__(self, K, N, seed, kind="llm", rows=ROWS):
        c = L.make_llm_case(K, N, G, rows, seed=seed, kind=kind)
        self.c, self.K, self.N = c, K, N
        special = np.concatenate([c["zero_cols"], c["ovf_low"], c["ovf_high"], c["cancel"]])
        self.cols = np.unique(np.concatenate([np.arange(0, N, 61), [0, 1, 7, 8, 15, 16, 255, 256, N - 9, N - 8, N - 1],
                                              special])).astype(np.int64)
        cols = self.cols
        self.bias = _t(c["bias"]) if c["bias"] is not None else None
        self.gemm = (_t(c["qweight"]), _t(c["scales"]), _t(c["qzeros"]))
        vw, vz, vs = O.pack_gemv(c["intweight"], c["zeros"], c["scales"], G)
        self.gemv = (_t(vw), _t(vs), _t(vz))
        fw, fs, fz = O.pack_gemv_fast(c["intweight"], c["zeros"], c["scales"], G)
        self.fast = (_t(fw), _t(fs), _t(fz))
        ng = K // G
        b = c["bias"][cols] if c["bias"] is not None else None
        self.sub = dict(w=c["w"][:, cols], scales=c["scales"][:, cols], group_size=G, bias=b)
        # GEMVFast: the stored tensors encode q s + sz, sz = fp16(-(z s)); its truth in fp64 on the sample
        qk = c["intweight"][:, cols].astype(np.float64)
        wf = qk * np.repeat(fs[:ng][:, cols].astype(np.float64), G, axis=0) + \
            np.repeat(fz[:ng][:, cols].astype(np.float64), G, axis=0)
        self.sub_fast = dict(w=wf, scales=fs[:ng][:, cols], group_size=G, bias=b)

    def forward(self, ext, layout, x, bias=True):
        return ext.linear_forward(layout, x, *getattr(self, layout), G, self.bias if bias else None)

    def family(self, layout, M, knobs=None):
        if layout == "gemm":
            return L.gemm_route_family(M, self.K, self.N, G, knobs)
        if layout == "gemv":
            return L.gemv_route_family(M, self.K, knobs)
        return L.fast_route_family(M, knobs)

    def check(self, y, x, layout, family, what, rows=None, bias=True):
        """y [M, N] (torch or numpy) against the truth of the rows `rows` of x (all when None)."""
        y = y.cpu().numpy() if torch.is_tensor(y) else y
        y = y.reshape(-1, self.N)[:, self.cols]
        x = np.asarray(x)
        if rows is not None:
            y, x = y[rows], x[rows]
        sub = dict(self.sub_fast if layout == "fast" else self.sub)
        if not bias:
            sub["bias"] = None
        hi = np.isin(self.cols, self.c["ovf_high"])
        if hi.any():
            y64 = x.astype(np.float64) @ sub["w"][:, hi].astype(np.float64)
            assert np.isinf(y[:, hi]).all() and (np.sign(y[:, hi].astype(np.float64)) == np.sign(y64)).all(), \
                f"{what}: an output beyond the fp16 range did not come back as inf of its sign"
            keep = ~hi
            y = y[:, keep]
            sub = dict(sub, w=sub["w"][:, keep], scales=sub["scales"][:, keep],
                       bias=sub["bias"][keep] if sub["bias"] is not None else None)
        r = L.check_forward(y, x, sub, family, what)
        key = (family, what.split(" M=")[0].split(": ")[-1])
        RATIOS[key] = max(RATIOS.get(key, 0.0), r)
        if family == "exact-dequant" and len(self.c["zero_cols"]):
            # W16 is exactly 0 there: every product and every partial sum is 0, the output is exactly the bias
            zc = np.isin(self.cols[~hi] if hi.any() else self.cols, self.c["zero_cols"])
            want = sub["bias"][zc] if sub["bias"] is not None else np.zeros(int(zc.sum()), dtype=np.float16)
            assert np.array_equal(y[:, zc], np.broadcast_to(want, (y.shape[0], int(zc.sum())))), \
                f"{what}: an all-zero column is not exactly the bias"
        return r


_CACHE: dict = {}


def _linear(K, N, seed, kind="llm"):
    key = (K, N, seed, kind)
    if key not in _CACHE:
        if len(_CACHE) >= 2:
            _CACHE.clear()
        _CACHE[key] = Linear(K, N, seed, kind)
    return _CACHE[key]


def _kn(knobs):
    return ",".join(f"knob{k}={v}" for k, v in knobs.items()) or "default knobs"


def _set_knobs(ext, knobs):
    prev = {k: ext.get_knob(k) for k in knobs}
    for k, v in knobs.items():
        ext.set_knob(k, v)
    return prev


def _workspace_is_zero(ext):
    torch.cuda.synchronize()
    for ws in ext._WS.values():
        assert int(ws.view(torch.int32).ne(0).sum()) == 0, "split-K scratch not restored"


# ------------------------------------------------------------------------------------------- dense linears
@pytest.mark.parametrize("name,K,N", SHAPES, ids=[s[0] for s in SHAPES])
def test_llm_data_all_layouts_all_m(ext, name, K, N):
    lin = _linear(K, N, seed=K % 97 + N % 89)
    x = lin.c["x"]
    for M in MS:
        xt = _t(x[:M])
        for layout in ("gemm", "gemv", "fast"):
            fam = lin.family(layout, M)
            lin.check(lin.forward(ext, layout, xt), x[:M], layout, fam, f"{name}: {layout} default M={M}")
    _workspace_is_zero(ext)


@pytest.mark.parametrize("knobs,Ms,what", ROUTES, ids=[r[2] for r in ROUTES])
@pytest.mark.parametrize("name,K,N", [SHAPES[1], SHAPES[3]], ids=[SHAPES[1][0], SHAPES[3][0]])
def test_llm_data_knob_routes(ext, name, K, N, knobs, Ms, what):
    lin = _linear(K, N, seed=K % 97 + N % 89)
    x = lin.c["x"]
    prev = _set_knobs(ext, knobs)
    try:
        for M in Ms:
            fam = lin.family("gemm", M, knobs)
            lin.check(lin.forward(ext, "gemm", _t(x[:M])), x[:M], "gemm", fam, f"{name}: gemm {what} M={M}")
        _workspace_is_zero(ext)
    finally:
        _set_knobs(ext, prev)


# ------------------------------------------------------------------------------------------ fp16 range edges
EDGE_ROUTES = [({}, (1, 2, 4, 5, 8, 16, 129, 300)), ({18: 1}, (1,)), ({5: 1}, (1, 8)), ({2: 0}, (1, 4)),
               ({21: 1}, (16, 64)), ({21: 2}, (16, 64)), ({19: 1}, (8, 64))]


@pytest.mark.parametrize("kind", ["overflow", "cancel"])
@pytest.mark.parametrize("name,K,N", [SHAPES[0], SHAPES[3]], ids=[SHAPES[0][0], SHAPES[3][0]])
def test_fp16_range_edges(ext, name, K, N, kind):
    """Exact outputs <= 65504 (1 - 2^-9) come back finite and within tolerance, >= 65520 (1 + 2^-8) as inf of their
    sign (the band between is not checked); columns whose K-halves are +-2^17 come back finite on every route,
    including the fp32-RED split-K and the small-M work cuts."""
    lin = _linear(K, N, seed=7, kind=kind)
    x = lin.c["x"]
    for knobs, Ms in EDGE_ROUTES:
        prev = _set_knobs(ext, knobs)
        try:
            for M in Ms:
                for layout in ("gemm", "gemv") if not knobs else ("gemm",):
                    fam = lin.family(layout, M, knobs)
                    y = lin.forward(ext, layout, _t(x[:M]), bias=False)
                    lin.check(y, x[:M], layout, fam, f"{name} {kind}: {layout} {kind} {_kn(knobs)} M={M}", bias=False)
        finally:
            _set_knobs(ext, prev)
    _workspace_is_zero(ext)


# ------------------------------------------------------------------------------------- non-finite activations
@pytest.mark.parametrize("layout", ["gemm", "gemv", "fast"])
def test_non_finite_rows_stay_in_their_rows(ext, layout):
    """One row with +inf on a massive channel, another with a NaN: those two rows are non-finite on every column
    (the reference gives +-inf or inf * 0 = NaN, the offset fold inf - inf), every other row is finite and within
    tolerance."""
    K, N = 4096, 4096
    lin = _linear(K, N, seed=K % 97 + N % 89)
    for M in (2, 3, 4, 5, 8, 16, 129):
        x = lin.c["x"][:M].copy()
        bad = [0, M - 1]
        x[0, lin.c["massive"][0]] = np.inf
        x[M - 1, 5] = np.nan
        y = lin.forward(ext, layout, _t(x)).cpu().numpy()
        assert not np.isfinite(y[bad]).any(), f"{layout} M={M}: a poisoned row has a finite output"
        good = [m for m in range(M) if m not in bad]
        if good:
            fam = lin.family(layout, M)
            lin.check(y, x, layout, fam, f"{layout} rows beside non-finite rows M={M}", rows=good)
    _workspace_is_zero(ext)


@pytest.mark.parametrize("layout,knobs,Ms", [
    ("gemm", {}, (1, 2, 3, 4, 5, 8, 16, 129)), ("gemm", {5: 1}, (1, 4, 8)), ("gemm", {2: 0}, (1, 4)),
    ("gemm", {18: 1}, (1,)), ("gemv", {}, (1, 2, 16)), ("fast", {}, (1, 2, 16)),
])
def test_activations_in_a_nan_filled_buffer(ext, layout, knobs, Ms):
    """x is a view into a NaN-filled buffer: the row-pitch gap and the rows before and after the M used are NaN.  A read
    outside the operand that reaches an FMA shows up even when it meets a zero weight."""
    K, N = 4096, 4096
    lin = _linear(K, N, seed=K % 97 + N % 89)
    prev = _set_knobs(ext, knobs)
    try:
        for M in Ms:
            buf = torch.full((M + 4, K + 64), float("nan"), dtype=torch.float16, device=_dev())
            xv = buf[2:2 + M, :K]
            xv.copy_(_t(lin.c["x"][:M]))
            y = lin.forward(ext, layout, xv)
            assert torch.isfinite(y).all(), f"{layout} {_kn(knobs)} M={M}: NaN from outside the operand"
            lin.check(y, lin.c["x"][:M], layout, lin.family(layout, M, knobs),
                      f"{layout} NaN-padded view {_kn(knobs)} M={M}")
    finally:
        _set_knobs(ext, prev)
    _workspace_is_zero(ext)


# ---------------------------------------------------------------------------------------------------- MoE
class Experts:
    """E experts over three distinct weights: two LLM-shaped ones and a dead one (every q equals its z, W = 0)."""
    DEAD = 2

    def __init__(self, K, N, seed):
        live = [L.make_llm_case(K, N, G, 1, seed=seed + i) for i in range(2)]
        dead = dict(live[0])
        dead["intweight"] = np.repeat(live[0]["zeros"], G, axis=0)
        dead["qweight"] = O.pack_gemm_words(dead["intweight"])
        dead["w"] = O.dequantize_gemm(dead["qweight"], dead["qzeros"], dead["scales"], G)
        assert not dead["w"].any()
        self.which = [0, 1, None, 0, 1, 0, 1, 0]                # expert e -> weights (None: dead)
        self.cases = [dead if i is None else live[i] for i in self.which]
        self.K, self.N = K, N
        self.cols = np.unique(np.concatenate([np.arange(0, N, 61), [0, 7, 8, 255, 256, N - 1]]))
        self.dev = tuple(_t(np.stack([c[k] for c in self.cases])) for k in ("qweight", "scales", "qzeros"))
        self.rng = np.random.default_rng(seed)

    def x(self, rows):
        x = self.rng.standard_normal((rows, self.K))
        x[:, 1000:1004] = np.array([300.0, -1200.0, 2500.0, -4000.0])   # massive channels, every row
        return x.astype(np.float16)

    def route(self, T, topk=2):
        ids = np.stack([self.rng.permutation(8)[:topk] for _ in range(T)]).astype(np.int32)
        ids[::3, 0] = self.DEAD                                  # some slots select the dead expert
        ids[::3, 1] = np.where(ids[::3, 1] == self.DEAD, 0, ids[::3, 1])
        tw = self.rng.random((T, topk)).astype(np.float32) + 0.1
        tw /= tw.sum(axis=1, keepdims=True)
        s, e, n = O.moe_align_block_size(ids, 16, 8)
        return ids, tw, _t(s), _t(np.where(e < 0, 0, e).astype(np.int32)), _t(np.array([n], dtype=np.int32))

    def check(self, ext, T, per_slot, mul, family, what):
        ids, tw, s_ids, e_ids, npost = self.route(T)
        x = self.x(T * 2 if per_slot else T)
        xt = _t(x).view(T, 2 if per_slot else 1, self.K)
        y = ext.grouped_gemm_forward(xt, *self.dev, _t(tw), s_ids, e_ids, npost, mul, 8).cpu().numpy()
        for t in range(T):
            for k in range(2):
                e = int(ids[t, k])
                c = self.cases[e]
                xr = x[t * 2 + k if per_slot else t][None, :]
                wgt = float(tw[t, k]) if mul else 1.0
                sub = dict(w=c["w"][:, self.cols].astype(np.float64) * wgt, group_size=G, bias=None,
                           scales=c["scales"][:, self.cols].astype(np.float64) * wgt)
                got = y[t, k, self.cols][None, :]
                r = L.check_forward(got, xr, sub, family, f"{what} T={T} token {t} slot {k} expert {e}")
                RATIOS[(family, what)] = max(RATIOS.get((family, what), 0.0), r)
                if e == self.DEAD and family == "exact-dequant":
                    assert not got.any(), f"{what}: the dead expert's output is not exactly 0"


MOE_OPS = [("gate_up", 4096, 28672, False), ("down", 14336, 4096, True), ("down N%256!=0", 14336, 3968, True)]


@pytest.mark.parametrize("op,K,N,per_slot", MOE_OPS, ids=[m[0] for m in MOE_OPS])
def test_grouped_gemm_llm_data(ext, op, K, N, per_slot):
    """Mixtral experts (8, top-2) with a dead expert: the ring kernel, the register-staged kernel (knob 12 = 2, and
    N % 256 != 0), and moe_tc_kernel at a prefill-sized T."""
    ex = Experts(K, N, seed=K + N)
    if N % 256 == 0:
        for T in (1, 5):
            ex.check(ext, T, per_slot, per_slot, "offset-fold", f"moe {op} ring")
        prev = _set_knobs(ext, {12: 2})
        try:
            ex.check(ext, 5, per_slot, per_slot, "offset-fold", f"moe {op} register-staged (knob 12 = 2)")
        finally:
            _set_knobs(ext, prev)
        ex.check(ext, 96, per_slot, per_slot, "exact-dequant", f"moe {op} moe_tc")
    else:
        ex.check(ext, 5, per_slot, per_slot, "offset-fold", f"moe {op} register-staged")
    _workspace_is_zero(ext)


# ---------------------------------------------------------------------------------------------- decode programs
_PROG_OPS: list = []


@pytest.mark.parametrize("replay", [False, True], ids=["fused", "knob14=1-replay"])
@pytest.mark.parametrize("M", [1, 2, 4, 8])
def test_program_of_independent_linears_llm_data(ext, M, replay):
    """The four Llama-3-8B linears in one DecodeProgram on LLM-shaped rows, fused (the stream / batched kernels,
    offset-fold) and replayed per op (knob 14 = 1, the per-op routes)."""
    from autoawq_b200.program import DecodeProgram

    if not _PROG_OPS:
        _CACHE.clear()
        _PROG_OPS.extend(Linear(K, N, seed=K % 97 + N % 89, rows=8) for _, K, N in SHAPES[:4])
    ops = _PROG_OPS
    prev = _set_knobs(ext, {14: 1 if replay else 0})
    try:
        prog = DecodeProgram(max_tokens=M)
        xs, ys = [], []
        for i, lin in enumerate(ops):
            xb = torch.zeros((M, lin.K), dtype=torch.float16, device=_dev())
            xs.append(xb)
            ys.append(prog.gemm_forward_cuda(xb, *lin.gemm, 8, bias=lin.bias if i % 2 else None))
        prog.build()
        fused = not replay and (M < 8 or max(lin.K for lin in ops) < 12288)
        assert prog.fused == fused, f"M={M}: fused={prog.fused}"
        for xb, lin in zip(xs, ops):
            xb.copy_(_t(lin.c["x"][:M]))
        prog.run()
        torch.cuda.synchronize()
        for i, (y, lin) in enumerate(zip(ys, ops)):
            fam = "offset-fold" if fused else lin.family("gemm", M)
            lin.check(y.view(M, -1), lin.c["x"][:M], "gemm", fam,
                      f"program {'fused' if fused else 'replayed'} op {i} M={M}", bias=bool(i % 2))
        if fused:
            rec = DecodeProgram.abort_record()
            assert rec[3] == 0, f"program kernel gave up waiting: code={rec[0]} op={rec[1]} cta={rec[2]}"
        prog.close()
    finally:
        _set_knobs(ext, prev)


def test_report_ratios():
    """Largest observed error / bound per family and route of this module's run."""
    for (fam, route), r in sorted(RATIOS.items()):
        print(f"RATIO {fam:14s} {r:.4f}  {route}")
