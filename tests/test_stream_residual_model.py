"""Executable model of residual reads in the stream decode program (csrc/program_stream.cuh, SpRes): when is it safe for
op i to read the published row of an older op j in its FINISH phase?

tests/test_stream_protocol_model.py covers the hand-off words polled at staging time.  A residual is read later, in the
finish of op i, one unit loop after the staging, and it sits in programs whose first op reads an external buffer (the
segment after attention starts with `o` reading the attention output).  Op j's row (j % 4) is published again by ops
j + 4, j + 8, ..., by whichever CTAs own its columns there; nothing but the staging polls orders CTAs against each other,
an op whose source is external waits for nobody, and an op that stages a SLICE of a row waits only for the CTAs that own
that slice.

The model replays random programs on a few CTAs with random and adversarial schedules: per op a staging step (poll the
words [off, off + K) of the source op's M rows until they carry its (run, op) stamp) and one finish step per owned column
and token row (read the residual word - it must still carry op j's stamp - then publish).  The CTA partition is the
kernel's: whole 16-column sets, set range [S c / G, S (c + 1) / G).  Ingredients: residual reads at finish time, ops with
external sources anywhere, sources that are slices of a row, batched rows (M > 1), several runs back to back (rows are
never cleared).  A write never replaces a newer stamp: whether an older op's store can land after a newer op's store to
the same word is a question of staging order (tests/test_stream_protocol_model.py); this model isolates residual reads.

Which programs fold is decided by the library itself: every random program is recorded as a b200awq_op_t list (fake
addresses, which the folding only compares) and handed to b200awq_program_plan, program_create's folding without any
CUDA call, with the model's CTA count.  With the library's window every accepted program is safe; with the window one
wider, accepted programs break.  Two Python variants of the rule show what its staging clause is for."""
import ctypes
import random

from autoawq_b200 import _cabi
from autoawq_b200._cabi import lib

ROWS = 4
OK = 0


# ------------------------------------------------------------------------------------------------ programs
def random_program(rng, n, d):
    """widths[i] (multiple of 16); src[i] = None (external) or (j, off, K): the columns [off, off + K) of op j's row,
    i - j <= 3 (the staging window); one residual: res[i] = j = i - d with equal widths."""
    widths = [rng.choice([16, 32, 48, 64]) for _ in range(n)]
    i = rng.randint(d, n - 1)
    j = i - d
    widths[i] = widths[j]
    src = [None]
    for m in range(1, n):
        if rng.random() < 0.3:
            src.append(None)
            continue
        s = rng.randint(max(0, m - 3), m - 1)
        if rng.random() < 0.6:
            src.append((s, 0, widths[s]))               # the whole row
        else:
            k = 16 * rng.randint(1, widths[s] // 16)
            off = 16 * rng.randint(0, (widths[s] - k) // 16)
            src.append((s, off, k))
    res = [None] * n
    res[i] = j
    return dict(widths=widths, src=src, res=res), i, j


def plan(prog, grid, window=0):
    """b200awq_program_plan of the program: (return code, kernel ops)."""
    widths, src, res = prog["widths"], prog["src"], prog["res"]
    base = [0x10000000]

    def buf():
        base[0] += 1 << 16
        return base[0]

    pub = []                               # the buffer each op's row publishes (the add's output when one folds in)
    ops = []
    for i, n_out in enumerate(widths):
        if src[i] is None:
            x, k = buf(), 16 * random.Random(i).randint(1, 4)
        else:
            j, off, k = src[i]
            x = pub[j] + 2 * off
        y = buf()
        ops.append(dict(kind=_cabi.OP_LINEAR_GEMM, M=1, K=k, N=n_out, group_size=k, ldx=k, x=x, qweight=buf(),
                        scales=buf(), qzeros=buf(), y=y))
        if res[i] is not None:
            out = buf()
            ops.append(dict(kind=_cabi.OP_ADD, M=1, K=n_out, x=y, weight=pub[res[i]], y=out))
            y = out
        pub.append(y)
    arr = (_cabi.Op * len(ops))()
    for c, o in zip(arr, ops):
        for f, v in o.items():
            setattr(c, f, v)
    kops = ctypes.c_int()
    rc = lib.b200awq_program_plan(arr, len(ops), 1, grid, window, ctypes.byref(kops))
    return rc, kops.value


def python_rule(prog, i, j, grid, count_slices=False, clause=True):
    """The rule restated, with the staging clause optionally weakened (slice waits counted) or dropped."""
    n, widths, src = len(prog["widths"]), prog["widths"], prog["src"]
    if widths[i] != widths[j] or not 1 <= i - j <= ROWS:
        return False
    k = j + ROWS
    while k <= i:
        k += ROWS
    if not clause or k >= n:
        return True
    for m in range(i + 1, k + 1):
        if src[m] is None:
            continue
        s, off, K = src[m]
        whole = off == 0 and K == widths[s]
        if s >= i and widths[s] // 16 >= grid and (whole or count_slices):
            return True
    return False


# ------------------------------------------------------------------------------------------------ the replay
def owned(width, grid, c):
    S = width // 16
    return range(16 * (S * c // grid), 16 * (S * (c + 1) // grid))


def simulate(prog, grid, M, runs, rng, victim=None):
    """Returns the residual violations: (op, column, the stamp the word carried instead of op j's)."""
    n, widths, src, res = len(prog["widths"]), prog["widths"], prog["src"], prog["res"]
    rows = [[[None] * max(widths) for _ in range(M)] for _ in range(ROWS)]   # word = (run, op) stamp
    bad = []

    def cta(c, run):                       # a generator of steps; a step yields False while it is blocked
        for i in range(n):
            if src[i] is not None:
                j, off, K = src[i]
                while True:
                    stamps = [rows[j % ROWS][m][col] for m in range(M) for col in range(off, off + K)]
                    if all(s == (run, j) for s in stamps):
                        break
                    if any(s is not None and s > (run, j) for s in stamps):
                        break              # a staging hazard: not what this model is about
                    yield False
            for col in owned(widths[i], grid, c):
                for m in range(M):
                    if res[i] is not None:
                        j = res[i]
                        while True:
                            s = rows[j % ROWS][m][col]
                            if s == (run, j):
                                break
                            if s is not None and s > (run, j):
                                bad.append((i, col, s))
                                break
                            yield False
                    w = rows[i % ROWS][m]
                    if w[col] is None or w[col] < (run, i):
                        w[col] = (run, i)
                    yield True

    for run in range(runs):                # runs are separate launches: every CTA finishes run r before run r + 1
        gens = [cta(c, run) for c in range(grid)]
        alive, spins = list(range(grid)), 0
        while alive:
            if victim in alive and len(alive) > 1 and rng.random() < 0.9:
                c = rng.choice([a for a in alive if a != victim])
            else:
                c = rng.choice(alive)
            try:
                progressed = next(gens[c])
            except StopIteration:
                alive.remove(c)
                continue
            spins = 0 if progressed else spins + 1
            assert spins <= 20000, "model deadlock"
    return bad


def _replay(accept, trials, seed, dists):
    """(accepted programs replayed, programs with a violation) over random programs the predicate accepts."""
    rng = random.Random(seed)
    tried = found = 0
    attempts = 0
    while tried < trials:
        attempts += 1
        assert attempts < 200 * trials, "the rule accepts almost nothing"
        d = rng.choice(dists)
        prog, i, j = random_program(rng, rng.randint(d + 1, 10), d)
        grid = rng.choice([2, 3, 5])
        if not accept(prog, i, j, grid):
            continue
        tried += 1
        if simulate(prog, grid, rng.choice([1, 2, 3]), runs=2, rng=rng, victim=rng.choice([None, 0, grid - 1])):
            found += 1
    return found


def _library_window():
    prog = dict(widths=[32] * 6, src=[None] + [(m - 1, 0, 32) for m in range(1, 6)], res=[None] * 6)
    w = 0
    for d in range(1, 8):
        p = dict(prog, res=[None] * 5 + [5 - d]) if d <= 5 else None
        if p is None or plan(p, grid=2)[0] != OK:
            break
        w = d
    return w


# ------------------------------------------------------------------------------------------------ tests
def test_library_window_is_the_row_rotation():
    assert _library_window() == ROWS


def test_library_rule_is_safe():
    accept = lambda p, i, j, g: plan(p, g)[0] == OK  # noqa: E731
    assert _replay(accept, trials=400, seed=1, dists=[1, 2, 3, 4]) == 0


def test_library_rule_widened_by_one_fails():
    accept = lambda p, i, j, g: plan(p, g, window=ROWS + 1)[0] == OK  # noqa: E731
    assert _replay(accept, trials=60, seed=2, dists=[ROWS + 1]) > 0


def test_library_rule_is_the_python_rule():
    rng = random.Random(4)
    for _ in range(600):
        d = rng.randint(1, ROWS)
        prog, i, j = random_program(rng, rng.randint(d + 1, 10), d)
        grid = rng.choice([2, 3, 5])
        assert (plan(prog, grid)[0] == OK) == python_rule(prog, i, j, grid), (prog, i, j, grid)


def test_without_the_staging_clause_every_distance_fails():
    for d in (1, 2, 3):
        accept = lambda p, i, j, g: python_rule(p, i, j, g, clause=False)  # noqa: E731
        assert _replay(accept, trials=300, seed=20 + d, dists=[d]) > 0, d


def test_a_wait_on_a_slice_does_not_order_every_cta():
    accept = lambda p, i, j, g: python_rule(p, i, j, g, count_slices=True) and not python_rule(p, i, j, g)  # noqa: E731
    assert _replay(accept, trials=150, seed=30, dists=[1, 2, 3, 4]) > 0


def test_llama_segment_shape():
    """o (external source) -> gate|up -> down + o's row -> qkv: residual two ops back, row 0 never republished."""
    prog = dict(widths=[64, 128, 64, 96], src=[None, (0, 0, 64), (1, 0, 128), (2, 0, 64)], res=[None, None, 0, None])
    assert plan(prog, grid=4) == (OK, 4)
    rng = random.Random(3)
    for _ in range(50):
        assert not simulate(prog, rng.choice([2, 3, 4]), rng.choice([1, 4]), runs=3, rng=rng, victim=rng.choice([None, 0]))
