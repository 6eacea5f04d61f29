"""Protocol-level simulation of the mbarrier / wgmma pipelines of the Hopper kernels: the swap-AB GEMM ring (csrc/gemm_tcgen05.cu,
decode_chain.cu, gemm_decode_fused.cu incl. NORM_IN, ts_encoder_fused.cu, gemm_w4.cu), the wgmma prefill attention
(csrc/attention.cu) and the wgmma attention backward (csrc/attention_bwd_wgmma.cu: dQ and dK/dV kernels).  The TMA producer and
the MMA warpgroup are transcribed as coroutines that perform the kernel's waits, arrivals, TMA issues, wgmma issues / commit
groups / wgmma_wait<N> and shared-memory writes in the kernel's order; a random scheduler interleaves them and completes the
asynchronous operations (TMA copies in any order, wgmma groups in issue order) at random later points.

What it checks, over many random schedules:
  * liveness -- every role terminates (a lost arrival or a wrong phase parity shows up as a deadlock);
  * every MMA reads the operand tiles it is meant to read, at issue time AND at completion time (a slot refilled too early --
    released before the wgmma group that reads it has been waited for -- or not yet filled, is a label mismatch);
  * the accumulator chain: every MMA adds to the result of the previous one.

mbarrier semantics modelled: arrival count, expect_tx / complete_tx byte accounting, phase parity with try_wait(parity)
(a fresh barrier passes a wait on parity 1).  wgmma_wait<N> returns once at most N committed groups are outstanding.
TEST INFRASTRUCTURE ONLY -- it pins the synchronisation design, not the data path.
"""
import random

import pytest


class MBar:
    def __init__(self, count):
        self.count, self.pending, self.tx, self.done = count, count, 0, 0

    def _check(self):
        if self.pending == 0 and self.tx == 0:
            self.done += 1
            self.pending = self.count

    def arrive(self):
        assert self.pending > 0, "more arrivals than the barrier was initialised for"
        self.pending -= 1
        self._check()

    def expect_tx(self, nbytes):
        self.tx += nbytes
        self.arrive()

    def complete_tx(self, nbytes):
        self.tx -= nbytes
        assert self.tx >= 0
        self._check()

    def ready(self, parity):
        return (self.done & 1) != parity


class Sim:
    def __init__(self, seed):
        self.rng = random.Random(seed)
        self.agents, self.async_ops, self.mma_queue = [], [], []
        self.mem = {}                                    # buffer name -> label of its current content

    def spawn(self, name, gen):
        self.agents.append([name, gen, None])            # [name, coroutine, pending wait predicate]

    # asynchronous engines ---------------------------------------------------------------------------------------------
    def tma(self, buf, label, bar, nbytes):
        self.async_ops.append(lambda: (self.mem.__setitem__(buf, label), bar.complete_tx(nbytes)))

    def mma(self, reads, write=None, chain=()):
        """reads: [(buffer, expected label)], write: (buffer, label).  Shared-memory operands are checked now and again at
        completion; ``chain`` = the accumulator this MMA adds to: the tensor core executes MMAs in issue order, so that
        dependency is checked at completion only."""
        for b, lab in reads:
            assert self.mem.get(b) == lab, f"MMA issued while {b} holds {self.mem.get(b)}, wanted {lab}"
        self.mma_queue.append(("mma", list(reads) + list(chain), write))

    def commit(self, bar):
        self.mma_queue.append(("commit", bar, None))

    def group(self):
        """wgmma.commit_group: the MMAs issued since the previous group form one group."""
        self.mma_queue.append(("group", None, None))

    def groups_pending(self):
        return sum(1 for kind, _, _ in self.mma_queue if kind == "group")

    def _step_mma(self):
        kind, a, b = self.mma_queue.pop(0)
        if kind == "group":
            return
        if kind == "commit":
            a.arrive()
            return
        for buf, lab in a:
            assert self.mem.get(buf) == lab, f"MMA completed after {buf} was refilled with {self.mem.get(buf)}, wanted {lab}"
        if b is not None:
            self.mem[b[0]] = b[1]

    def run(self, max_steps=200000):
        for _ in range(max_steps):
            choices = []
            for ag in self.agents:
                if ag[2] is None or ag[2]():
                    choices.append(("agent", ag))
            if self.async_ops:
                choices.append(("async", None))
            if self.mma_queue:
                choices.append(("mma", None))
            if not choices:
                if all(ag[1] is None for ag in self.agents):
                    return
                blocked = [ag[0] for ag in self.agents if ag[1] is not None]
                raise AssertionError(f"deadlock: {blocked} blocked with no asynchronous work outstanding")
            kind, ag = self.rng.choice(choices)
            if kind == "async":
                self.async_ops.pop(self.rng.randrange(len(self.async_ops)))()
            elif kind == "mma":
                self._step_mma()
            else:
                try:
                    ag[2] = next(ag[1])                  # the coroutine yields its next wait predicate (or None to just yield)
                except StopIteration:
                    ag[1], ag[2] = None, (lambda: False)
            self.agents = [a for a in self.agents if a[1] is not None] + [a for a in self.agents if a[1] is None]
            if all(a[1] is None for a in self.agents) and not self.async_ops and not self.mma_queue:
                return
        raise AssertionError("simulation did not finish")


def wait(bar, parity):
    return lambda: bar.ready(parity)


def wgmma_wait(s, n):
    return lambda: s.groups_pending() <= n


# ====================================================================================================================== swap-AB GEMM ring
def sim_gemm_ring(nkb, stages, seed, norm_in=False):
    """Producer: weight tile (and, unless NORM_IN, the token tile) of K block i into slot i % stages once the slot is released.
    MMA warpgroup: per block -- (NORM_IN: write the token tile into the slot itself) -- wait full, issue, commit a group,
    wgmma_wait<1>, release the PREVIOUS block's slot; after the loop wgmma_wait<0> and release the last slot."""
    s = Sim(seed)
    full, empty = [MBar(1) for _ in range(stages)], [MBar(1) for _ in range(stages)]
    for st in range(stages):
        s.mem[f"A{st}"], s.mem[f"B{st}"] = None, None
    s.mem["acc"] = ("acc", -1)

    def producer():
        for i in range(nkb):
            st = i % stages
            yield wait(empty[st], ((i // stages) & 1) ^ 1)
            full[st].expect_tx(1 if norm_in else 2)
            s.tma(f"A{st}", ("A", i), full[st], 1)
            if not norm_in:
                s.tma(f"B{st}", ("B", i), full[st], 1)
            yield None

    def mma():
        for i in range(nkb):
            st = i % stages
            if norm_in:                                   # slot st was last read by block i - stages: waited for below
                s.mem[f"B{st}"] = ("B", i)
                yield None                                # named barrier of the four warps
            yield wait(full[st], (i // stages) & 1)
            s.mma([(f"A{st}", ("A", i)), (f"B{st}", ("B", i))], ("acc", ("acc", i)), chain=[("acc", ("acc", i - 1))])
            s.group()
            yield wgmma_wait(s, 1)
            if i > 0:
                empty[(i - 1) % stages].arrive()
            yield None
        yield wgmma_wait(s, 0)
        if nkb > 0:
            empty[(nkb - 1) % stages].arrive()
        assert s.mem["acc"] == ("acc", nkb - 1)

    s.spawn("tma", producer())
    s.spawn("mma", mma())
    s.run()


# ====================================================================================================================== attention kernels
def sim_attention(n, fixed, ring, phase1, phase2, seed, acc_names):
    """The wgmma attention kernels: `fixed` tiles land once on one barrier, `ring` tiles per item on a two-stage ring.  Per item the
    warpgroup issues the phase-1 MMAs (both operands in shared memory: S / dP), waits for them (wgmma_wait<0>), runs the softmax in
    registers, issues the phase-2 MMAs (register A operand, a ring tile as B: O, dQ, dV, dK) into the accumulators, waits again and
    only then releases the ring slot."""
    s = Sim(seed)
    fix, full, empty = MBar(1), [MBar(1), MBar(1)], [MBar(1), MBar(1)]
    for f in fixed:
        s.mem[f] = None
    for st in range(2):
        for r in ring:
            s.mem[f"{r}{st}"] = None
    for a in acc_names:
        s.mem[a] = (a, -1)

    def tile(name, st):
        return name if name in fixed else f"{name}{st}"

    def label(name, j):
        return name if name in fixed else (name, j)

    def producer():
        fix.expect_tx(len(fixed))
        for f in fixed:
            s.tma(f, f, fix, 1)
        for j in range(n):
            st = j & 1
            yield wait(empty[st], ((j >> 1) & 1) ^ 1)
            full[st].expect_tx(len(ring))
            for r in ring:
                s.tma(f"{r}{st}", (r, j), full[st], 1)
            yield None

    def mma():
        yield wait(fix, 0)
        for j in range(n):
            st = j & 1
            yield wait(full[st], (j >> 1) & 1)
            for x, y in phase1:
                s.mma([(tile(x, st), label(x, j)), (tile(y, st), label(y, j))])
            s.group()
            yield wgmma_wait(s, 0)
            yield None                                    # softmax / dS in registers
            for b_op, acc in phase2:
                s.mma([(tile(b_op, st), label(b_op, j))], (acc, (acc, j)), chain=[(acc, (acc, j - 1))])
            s.group()
            yield wgmma_wait(s, 0)
            empty[st].arrive()
            yield None
        for acc in acc_names:
            assert s.mem[acc] == (acc, n - 1)

    s.spawn("tma", producer())
    s.spawn("mma", mma())
    s.run()


def sim_dq(nt, seed):
    sim_attention(nt, ["Q", "dO"], ["K", "V"], [("Q", "K"), ("dO", "V")], [("K", "dQ")], seed, ["dQ"])


def sim_dkv(n_iter, seed):
    sim_attention(n_iter, ["K", "V"], ["Q", "dO"], [("K", "Q"), ("V", "dO")], [("dO", "dV"), ("Q", "dK")], seed, ["dV", "dK"])


def sim_fused_norm_in(nkb, stages, seed):
    sim_gemm_ring(nkb, stages, seed, norm_in=True)


@pytest.mark.parametrize("nt", [1, 2, 3, 6])
def test_dq_pipeline(nt):
    for seed in range(60):
        sim_dq(nt, seed)


@pytest.mark.parametrize("n_iter", [1, 2, 5, 8])
def test_dkv_pipeline(n_iter):
    for seed in range(60):
        sim_dkv(n_iter, seed)


@pytest.mark.parametrize("nkb,stages", [(1, 3), (3, 3), (7, 3), (12, 2), (11, 4)])
def test_fused_decode_norm_in_pipeline(nkb, stages):
    for seed in range(60):
        sim_fused_norm_in(nkb, stages, seed)


@pytest.mark.parametrize("nkb,stages", [(1, 2), (2, 2), (5, 3), (12, 4)])
def test_gemm_ring_pipeline(nkb, stages):
    for seed in range(60):
        sim_gemm_ring(nkb, stages, seed)


@pytest.mark.parametrize("nt", [1, 2, 5])
def test_attention_forward_pipeline(nt):
    for seed in range(60):
        sim_attention(nt, ["Q"], ["K", "V"], [("Q", "K")], [("V", "O")], seed, ["O"])


def test_the_simulator_catches_a_missing_wait():
    """Self-check: a warpgroup that releases the slot of block i right after issuing its MMAs (no wgmma_wait before the arrive)
    lets the producer refill it under MMAs that still read it; the simulation must report that on some schedule."""
    def broken(seed, stages=2, nkb=6):
        s = Sim(seed)
        full, empty = [MBar(1) for _ in range(stages)], [MBar(1) for _ in range(stages)]
        for st in range(stages):
            s.mem[f"A{st}"] = None
        s.mem["acc"] = ("acc", -1)

        def producer():
            for i in range(nkb):
                st = i % stages
                yield wait(empty[st], ((i // stages) & 1) ^ 1)
                full[st].expect_tx(1)
                s.tma(f"A{st}", ("A", i), full[st], 1)
                yield None

        def mma():
            for i in range(nkb):
                st = i % stages
                yield wait(full[st], (i // stages) & 1)
                s.mma([(f"A{st}", ("A", i))], ("acc", ("acc", i)), chain=[("acc", ("acc", i - 1))])
                s.group()
                empty[st].arrive()                       # BUG: no wgmma_wait before the release
                yield None
            yield wgmma_wait(s, 0)

        s.spawn("tma", producer())
        s.spawn("mma", mma())
        s.run()

    caught = 0
    for seed in range(200):
        try:
            broken(seed)
        except AssertionError:
            caught += 1
    assert caught > 0
