"""Executable model of the small-M tensor-core kernel's pipeline protocol (csrc/gemm_tc.cu: gemm_tcq_kernel), run on
the CPU.  The kernel's four kinds of warps talk through mbarrier rings only - packed stages (Q-TMA -> the producer
warps), A stages (producers -> the consumer warpgroups), activation stages (X-TMA -> consumers) - and each of the two
consumer warpgroups (independent roles, one arrival per warp) releases a stage only after the wgmma group that read it
has retired (`wgmma.wait_group 1` after issuing the next group, `wait_group 0` at the end of a segment).  Every ring index / phase-parity expression of the device code is
restated here verbatim.  Random interleavings of the roles (and of the asynchronous agents: TMA landings, tensor-core
execution) check

  * liveness: every role finishes (no lost wake-up, no wait on a parity that never comes);
  * safety: a stage is never overwritten before its last reader has read it, and every reader sees exactly the step it
    expects (packed stage d -> both k-steps of the pair, A stage of k-step s -> the MMA of k-step s, X stage likewise),
    also across ring wrap-arounds, several segments per CTA and one-pair ranges;
  * the accumulators the epilogue reads hold exactly the k-steps of the segment, once each.

The model knows nothing about CUDA: it pins the index arithmetic, which is where such kernels break.  (The real
kernel's own tests are tests/test_gpu_parity.py::test_small_m_*.)"""
import random

import pytest


class Mbar:
    """mbarrier with a pending-arrival count per phase; wait(parity) passes once the latest phase of that parity is
    complete (a fresh barrier lets parity 1 through: the `phase ^ 1` idiom of the producers)."""

    def __init__(self, count):
        self.count, self.arrivals, self.done = count, 0, 0   # done = completed phases

    def arrive(self):
        self.arrivals += 1
        assert self.arrivals <= self.count, "more arrivals than the barrier was initialised for"
        if self.arrivals == self.count:
            self.arrivals, self.done = 0, self.done + 1

    def passed(self, parity):
        return (self.done & 1) != parity


class Sim:
    def __init__(self, NS, NX, NQ, ranges, KP, seed, empty_count=8):
        self.NS, self.NX, self.NQ, self.KP = NS, NX, NQ, KP
        self.t_begin, self.t_end = ranges
        self.rng = random.Random(seed)
        self.full = [Mbar(8) for _ in range(NS)]          # 8 producer warps (modelled as 1 agent x 8 arrivals)
        self.empty = [Mbar(empty_count) for _ in range(NS)]   # 8 consumer warps: 4 per warpgroup
        self.xfull = [Mbar(2) for _ in range(NX)]         # expect_tx arrival + "bytes landed"
        self.xempty = [Mbar(empty_count) for _ in range(NX)]
        self.qfull = [Mbar(2) for _ in range(NQ)]
        self.qempty = [Mbar(8) for _ in range(NQ)]
        self.q_data = [None] * NQ                          # content tags: what a stage currently holds
        self.a_data = [None] * NS
        self.x_data = [None] * NX
        self.acc = [[], []]                                # per consumer warpgroup: k-steps of its retired MMAs
        self.async_ops = []                                # pending asynchronous actions (TMA landings, MMA execution)
        self.drained = []                                  # (segment, steps) seen by the epilogue

    # ---- segment walk shared by all roles (device: nt / d0 / d1 from t)
    def segments(self):
        t, out = self.t_begin, []
        while t < self.t_end:
            nt = t // self.KP
            d0 = t - nt * self.KP
            d1 = self.KP if self.KP - d0 < self.t_end - t else d0 + (self.t_end - t)
            out.append((nt, d0, d1))
            t += d1 - d0
        return out

    # ---- roles as generators: `yield cond` blocks until cond() is true
    def q_tma(self):
        qs, qph = 0, 0
        for nt, d0, d1 in self.segments():
            for d in range(d0, d1):
                yield lambda qs=qs, qph=qph: self.qempty[qs].passed(qph ^ 1)
                self.qfull[qs].arrive()                                    # arrive.expect_tx
                self.async_ops.append(("land_q", qs, (nt, d)))
                qs += 1
                if qs == self.NQ:
                    qs, qph = 0, qph ^ 1

    def x_tma(self):
        xs, xph = 0, 0
        for nt, d0, d1 in self.segments():
            for s in range(2 * d0, 2 * d1):
                yield lambda xs=xs, xph=xph: self.xempty[xs].passed(xph ^ 1)
                self.xfull[xs].arrive()
                self.async_ops.append(("land_x", xs, (nt, s)))
                xs += 1
                if xs == self.NX:
                    xs, xph = 0, xph ^ 1

    def producer(self):
        qs, stage, qph, phase = 0, 0, 0, 0
        for nt, d0, d1 in self.segments():
            for d in range(d0, d1):
                yield lambda qs=qs, qph=qph: self.qfull[qs].passed(qph)
                got = self.q_data[qs]                                      # fetch: LDS of both halves of the stage
                assert got == (nt, d), f"packed stage {qs} holds {got}, expected {(nt, d)}"
                for h in range(2):
                    yield lambda stage=stage, phase=phase: self.empty[stage].passed(phase ^ 1)
                    self.a_data[stage] = (nt, 2 * d + h)                   # dequantised tile of k-step 2 d + h
                    for _ in range(8):
                        self.full[stage].arrive()
                        if h == 1:
                            self.qempty[qs].arrive()
                    stage += 1
                    if stage == self.NS:
                        stage, phase = 0, phase ^ 1
                qs += 1
                if qs == self.NQ:
                    qs, qph = 0, qph ^ 1

    def pending_mma(self, wg):
        return sum(1 for op in self.async_ops if op[0] == "mma" and op[1] == wg)

    def consumer(self, wg):
        """Consumer warpgroup wg (4 warps, one arrival each): its own wgmma groups, its own half of every A stage."""
        stage, xs, phase, xph = 0, 0, 0, 0
        for it, (nt, d0, d1) in enumerate(self.segments()):
            self.acc[wg] = []
            prev = None
            for s in range(2 * d0, 2 * d1):
                yield lambda xs=xs, xph=xph: self.xfull[xs].passed(xph)
                yield lambda stage=stage, phase=phase: self.full[stage].passed(phase)
                # issue + commit: the tensor core reads the operands LATER (asynchronously)
                self.async_ops.append(("mma", wg, stage, xs, (nt, s)))
                yield lambda: self.pending_mma(wg) <= 1                   # wgmma.wait_group 1
                if prev is not None:
                    for _ in range(4):
                        self.empty[prev[0]].arrive()
                        self.xempty[prev[1]].arrive()
                prev = (stage, xs)
                stage += 1
                if stage == self.NS:
                    stage, phase = 0, phase ^ 1
                xs += 1
                if xs == self.NX:
                    xs, xph = 0, xph ^ 1
            yield lambda: self.pending_mma(wg) == 0                       # wgmma.wait_group 0
            if prev is not None:
                for _ in range(4):
                    self.empty[prev[0]].arrive()
                    self.xempty[prev[1]].arrive()
            want = [(nt, s) for s in range(2 * d0, 2 * d1)]
            assert sorted(self.acc[wg]) == want, f"segment {it}, warpgroup {wg}: accumulators hold {self.acc[wg]}"
            self.drained.append((it, wg, list(self.acc[wg])))

    # ---- asynchronous agents: the tensor core executes each warpgroup's MMAs in issue order (the two warpgroups
    # independently); TMA landings of one ring may complete in any order relative to other rings - pick any op that is
    # first of its (kind, ring or warpgroup) queue
    def step_async(self):
        if not self.async_ops:
            return False
        firsts, seen = [], set()
        for i, op in enumerate(self.async_ops):
            key = (op[0], op[1])
            if key not in seen:
                seen.add(key)
                firsts.append(i)
        op = self.async_ops.pop(self.rng.choice(firsts))
        if op[0] == "land_q":
            _, qs, tag = op
            self.q_data[qs] = tag
            self.qfull[qs].arrive()
        elif op[0] == "land_x":
            _, xs, tag = op
            self.x_data[xs] = tag
            self.xfull[xs].arrive()
        else:
            _, wg, stage, xs, want = op
            assert self.a_data[stage] == want, f"MMA {wg}: A stage {stage} holds {self.a_data[stage]}, expected {want}"
            assert self.x_data[xs] == want, f"MMA {wg}: X stage {xs} holds {self.x_data[xs]}, expected {want}"
            self.acc[wg].append(want)
        return True

    def run(self):
        roles = {"q": self.q_tma(), "x": self.x_tma(), "p": self.producer(), "c0": self.consumer(0), "c1": self.consumer(1)}
        waiting = {}
        for name, gen in list(roles.items()):
            try:
                waiting[name] = next(gen)
            except StopIteration:
                del roles[name]
        idle = 0
        while roles:
            progressed = False
            choices = list(roles) + ["async"] * 3
            self.rng.shuffle(choices)
            for name in choices:
                if name == "async":
                    progressed |= self.step_async()
                    continue
                if name in roles and waiting[name]():
                    try:
                        waiting[name] = roles[name].send(None)
                    except StopIteration:
                        del roles[name]
                    progressed = True
            idle = 0 if progressed else idle + 1
            assert idle < 3, f"deadlock: {sorted(roles)} blocked, {len(self.async_ops)} async ops pending"
        while self.step_async():
            pass
        assert len(self.drained) == 2 * len(self.segments())


CONFIGS = [
    # NS, NX, NQ   (BT <= 16: 4 / 16 / 14; BT = 64: 4 / 8 / 11; BT = 128: 4 / 4 / 11) + small rings that wrap constantly
    (4, 16, 14), (4, 8, 11), (4, 4, 11), (4, 2, 2), (2, 2, 3),
]
RANGES = [
    # (t_begin, t_end), KP: one segment, straddling segments, whole tiles, three segments (buffer recycling), one pair
    ((0, 32), 32), ((20, 75), 32), ((64, 128), 32), ((30, 100), 32), ((7, 8), 9), ((5, 40), 9), ((0, 3), 1),
]


@pytest.mark.parametrize("NS,NX,NQ", CONFIGS)
@pytest.mark.parametrize("rng_range,KP", RANGES)
def test_pipeline_protocol_random_interleavings(NS, NX, NQ, rng_range, KP):
    for seed in range(6):
        Sim(NS, NX, NQ, rng_range, KP, seed).run()


def test_model_detects_a_missing_release():
    """The model is not vacuous: without the producers' wait for `empty` an A stage is overwritten before its MMA ran."""

    class Broken(Sim):
        def producer(self):
            for cond in Sim.producer(self):
                yield cond if "empty" not in cond.__code__.co_names else (lambda: True)

    caught = 0
    for seed in range(20):
        try:
            Broken(2, 16, 14, (0, 64), 32, seed).run()
        except AssertionError:
            caught += 1
    assert caught > 0


def test_model_detects_a_barrier_count_of_one_warpgroup():
    """With `empty` / `xempty` initialised for one warpgroup's 4 arrivals instead of both warpgroups' 8, the faster
    warpgroup frees a stage the other one may still be reading."""
    caught = 0
    for seed in range(40):
        try:
            Sim(2, 2, 3, (0, 64), 32, seed, empty_count=4).run()
        except AssertionError:
            caught += 1
    assert caught > 0
