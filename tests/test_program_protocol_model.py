"""Executable model of the decode-program kernel's hand-off and row-reclamation protocol (csrc/program.cu):
random interleavings of the per-CTA agents (consumers, duty warp) over the shared state the kernel uses - packed rows
with a per-column tile count, the staged[] / zeroed[] counters, the per-CTA red_ok / staged_op flags - checking

  * safety: a push into row (op % 4) never lands before every CTA has zeroed its slice after op - 4, a slice is never
    zeroed while some agent still has to read that row, a reader never accepts a column before all its tiles arrived;
  * liveness: every schedule terminates (no deadlock, no lost wake-up), and all rows are zero at exit.

The deadlock found on the GPU is reproduced by `lane0_publishes_early` (the duty warp's lane 0 published staged[i]
before the warp's other lanes had finished polling row i-1: another CTA then zeroed the row under them).
`flag_only_row_clean` models consumers that rely on the duty warp's red_ok flag alone; the model shows that variant
is live too (all duty warps are within one iteration of each other because each waits for staged[i] of ALL CTAs), so
the kernel's direct check of zeroed[] is a defensive fall-back, not a fix.  The model is hand-written from the
kernel; it guards the protocol's logic, not the CUDA code."""
import random

import pytest

ROWS = 4


class Abort(Exception):
    pass


def run(n_cta, n_ops, cols_per_slice, seed, lane0_publishes_early=False, flag_only_row_clean=False, max_steps=200000):
    rng = random.Random(seed)
    ncol = n_cta * cols_per_slice                     # every op has ncol columns; CTA b's slice = its cols_per_slice
    tiles_per_col = n_cta                             # every CTA contributes one "tile" to every column
    rows = [[0] * ncol for _ in range(ROWS)]          # tile counts (the sum itself is irrelevant to the protocol)
    zero_gen = [[0] * ncol for _ in range(ROWS)]      # how many times a column was zeroed
    staged = [0] * (n_ops + 1)
    zeroed = [0] * (n_ops + 1)
    red_ok = [0] * n_cta
    staged_op = [0] * n_cta

    # ---- agents as generators: every `yield` is a point where another agent may run ---------------------
    def consumer(b):
        for op in range(n_ops):
            if op > 0:
                prev = rows[(op - 1) % ROWS]
                for c in range(ncol):                                   # stage: poll the previous op's row
                    while prev[c] != tiles_per_col:
                        assert prev[c] < tiles_per_col, "column over-complete: stale data under a new op"
                        yield
                staged_op[b] = op
                yield
            # tile loop ... then: row clean?
            if op > 0:
                while red_ok[b] < op:
                    if not flag_only_row_clean and (op < ROWS or zeroed[op - ROWS] >= n_cta):
                        break
                    yield
            if op >= ROWS:
                assert zeroed[op - ROWS] >= n_cta, f"push of op {op} before row was recycled"
            cur = rows[op % ROWS]
            for c in range(ncol):                                       # push one tile into every column
                cur[c] += 1
                if rng.random() < 0.3:
                    yield
            yield

    def duty(b):
        rk = 0

        def advance():
            nonlocal rk
            r = rk
            while r + 1 < n_ops and (r + 1 < ROWS or zeroed[r + 1 - ROWS] >= n_cta):
                r += 1
            rk = r
            red_ok[b] = r

        for i in range(1, n_ops + 1):
            advance()
            prev = rows[(i - 1) % ROWS]
            lo, hi = b * cols_per_slice, (b + 1) * cols_per_slice
            # the columns a duty warp READS (its slice of the fp16 output and of the SiLU*mul output) are not the
            # columns it ZEROES (its slice of the accumulator row): model that with the neighbour's slice
            nb = (b + 1) % n_cta
            lanes = list(range(lo, hi))
            if i < n_ops:
                lanes += list(range(nb * cols_per_slice, (nb + 1) * cols_per_slice))
            published = False
            for k, c in enumerate(lanes):                               # the warp's lanes poll their columns
                if lane0_publishes_early and k == 1 and i < n_ops and not published:
                    while staged_op[b] < i:
                        yield
                    staged[i] += 1                                      # BUG: lane 0 ran ahead of the other lanes
                    published = True
                while prev[c] != tiles_per_col:
                    yield
                yield                                                   # lanes do not finish together
            if i < n_ops:
                if not published:
                    while staged_op[b] < i:
                        yield
                    staged[i] += 1
                advance()
                while staged[i] < n_cta:
                    yield
                for c in range(lo, hi):                                 # recycle the slice of row i-1
                    prev[c] = 0
                    zero_gen[(i - 1) % ROWS][c] += 1
                    if rng.random() < 0.2:
                        yield
                zeroed[i - 1] += 1
                yield
            else:
                # epilogue: every duty warp reads only its own slice of the last row, then zeroes exactly that slice
                for c in range(lo, hi):
                    prev[c] = 0

    agents = [consumer(b) for b in range(n_cta)] + [duty(b) for b in range(n_cta)]
    live = list(range(len(agents)))
    steps = 0
    while live:
        steps += 1
        if steps > max_steps:
            raise Abort(f"no progress after {max_steps} steps: deadlock / lost wake-up (seed {seed})")
        k = rng.choice(live)
        try:
            next(agents[k])
        except StopIteration:
            live.remove(k)
    assert all(v == 0 for r in rows for v in r), "rows not clean at exit"
    return steps


@pytest.mark.parametrize("seed", range(25))
def test_protocol_random_schedules(seed):
    run(n_cta=3 + seed % 3, n_ops=9 + seed % 5, cols_per_slice=2, seed=seed)


def test_protocol_catches_the_lane0_bug():
    """Publishing staged[i] before the warp's other lanes finished polling lets another CTA zero the row under them:
    they then wait for ever (what the kernel's abort record showed on the GPU)."""
    hit = 0
    for seed in range(40):
        try:
            run(4, 10, 3, seed, lane0_publishes_early=True, max_steps=60000)
        except (Abort, AssertionError):
            hit += 1
    assert hit > 0


@pytest.mark.parametrize("seed", range(10))
def test_protocol_flag_only_variant_is_live_too(seed):
    run(4, 12, 2, seed, flag_only_row_clean=True)
