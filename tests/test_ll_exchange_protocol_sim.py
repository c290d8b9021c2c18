"""CPU: randomised-schedule simulation of the barrier-free push exchange (csrc/allreduce_ll.cu, "LL" protocol).

There are no barriers in that kernel: every 8-byte unit that crosses NVLink carries its own epoch tag and receivers poll the
data.  What must hold for every interleaving of ranks and CTAs and every delivery order of the pushed units:
  * a receiver only ever consumes units of THIS exchange (tag match => payload of this exchange, both halves of a line),
  * a pushed unit never overwrites a line its receiver has not consumed yet (receive buffers are reused every second exchange:
    slot = k % 2),
  * the GEMM that follows sees every row of x_out from this exchange,
  * nobody waits forever - PROVIDED every CTA can eventually run alongside the peer CTAs it waits for.  The simulator dispatches
    CTAs in any order, so it needs the whole grid resident and shows why.  The kernel's grid of 2 CTAs per SM is not always one
    wave (at 512 threads one CTA fits per SM); it relies on CTA c waiting only for CTA c of each peer and on CTAs being
    dispatched in blockIdx order (csrc/allreduce_ll.cu).
The model: per rank a stream (GEMM -> exchange kernel -> consumer GEMM), per CTA a state machine that mirrors the kernel's three
phases, a network that delivers every pushed half-line independently after an arbitrary delay and in arbitrary order, all under
a seeded random scheduler.  It validates the protocol the kernel implements, not the CUDA code (tests/test_exchange_kernels_gpu.py
holds the kernel to a bit-exact restatement on one GPU, tests/test_tp_gpu.py runs it across GPUs)."""
import random

import pytest


class Violation(Exception):
    pass


class Line:
    """One 16-byte LL line = two self-validating halves {payload version, tag}."""
    __slots__ = ("tag", "ver", "consumed")

    def __init__(self):
        self.tag = [0, 0]; self.ver = [-1, -1]; self.consumed = True


class LlSim:
    def __init__(self, n, tokens, exchanges, resident, seed=0, slots=2, tokens_per_exchange=None):
        self.n, self.K, self.S, self.resident = n, exchanges, slots, resident
        self.Ts = tokens_per_exchange or [tokens] * exchanges          # T may change from one exchange to the next (eager steps)
        self.maxT = max(self.Ts)
        self.rows_per_rank = (self.maxT + n - 1) // n
        self.rng = random.Random(seed)
        self.partial = [[{"ver": -1, "dirty": False} for _ in range(slots)] for _ in range(n)]
        self.rs = [[[[Line() for _ in range(self.rows_per_rank)] for _ in range(n)] for _ in range(slots)] for _ in range(n)]  # [dst][slot][src][idx]
        self.ag = [[[Line() for _ in range(self.maxT)] for _ in range(slots)] for _ in range(n)]                               # [dst][slot][t]
        self.xout = [[-1] * self.maxT for _ in range(n)]
        self.epoch = [[0] * slots for _ in range(n)]
        self.done = [[0] * slots for _ in range(n)]
        self.net = []                                   # in-flight half-line stores: (line, half, tag, ver)
        self.streams = [self._stream(r) for r in range(n)]
        self.finished = [False] * n

    def grid(self, T):
        return T                                        # one CTA per row; `resident` decides how many run at once

    def _stream(self, r):
        for k in range(self.K):
            slot, T = k % self.S, self.Ts[k]
            yield [self._gemm(r, k, slot)]
            yield [self._cta(r, k, slot, c, T) for c in range(self.grid(T))]
            yield [self._consume(r, k, T)]

    def _gemm(self, r, k, slot):
        self.partial[r][slot]["dirty"] = True
        yield
        self.partial[r][slot].update(ver=k, dirty=False)
        yield

    def _read_partial(self, r, slot, k):
        p = self.partial[r][slot]
        if p["dirty"] or p["ver"] != k:
            raise Violation(f"rank {r} reads its partial slot {slot} for exchange {k}: {p}")

    def _push(self, line, tag, ver):
        # the two halves of a 16-byte store may land separately and late
        self.net.append((line, 0, tag, ver)); self.net.append((line, 1, tag, ver))

    def _deliver(self):
        line, half, tag, ver = self.net.pop(self.rng.randrange(len(self.net)))
        if half == 0 and not line.consumed and line.tag[0] != tag:
            raise Violation(f"a push of tag {tag} overwrites a line of tag {line.tag} that its receiver has not consumed")
        line.tag[half], line.ver[half] = tag, ver
        if line.tag[0] == line.tag[1]:
            line.consumed = False

    def _poll(self, line, e, k):
        while not (line.tag[0] == e and line.tag[1] == e):
            yield "wait"
        if line.ver != [k, k]:
            raise Violation(f"tag {e} matched but the payload is of exchange {line.ver}, expected {k}")
        line.consumed = True

    def _cta(self, r, k, slot, c, T):
        e = self.epoch[r][slot] + 1
        yield
        n, t = self.n, c
        # phase 1
        if t % n != r:
            self._read_partial(r, slot, k)
            self._push(self.rs[t % n][slot][r][t // n], e, k)
            yield
        # phase 2
        if t % n == r:
            for src in range(n):
                if src == r:
                    self._read_partial(r, slot, k)
                else:
                    yield from self._poll(self.rs[r][slot][src][t // n], e, k)
                yield
            self.xout[r][t] = k
            for i in range(1, n):
                self._push(self.ag[(r + i) % n][slot][t], e, k)
                yield
        else:
            # phase 3
            yield from self._poll(self.ag[r][slot][t], e, k)
            self.xout[r][t] = k
            yield
        self.done[r][slot] += 1
        if self.done[r][slot] == self.grid(T):
            self.done[r][slot] = 0
            self.epoch[r][slot] = e
        yield

    def _consume(self, r, k, T):
        if any(v != k for v in self.xout[r][:T]):
            raise Violation(f"rank {r} consumes x_out of exchange {k} but holds versions {sorted(set(self.xout[r][:T]))}")
        yield

    def run(self, max_steps=3_000_000):
        pending = [[] for _ in range(self.n)]
        active = [[] for _ in range(self.n)]
        idle = 0
        for _ in range(max_steps):
            if all(self.finished):
                return
            if self.net and self.rng.random() < 0.3:
                self._deliver(); idle = 0
                continue
            r = self.rng.randrange(self.n)
            if self.finished[r]:
                continue
            if not active[r] and not pending[r]:
                try:
                    pending[r] = list(next(self.streams[r]))
                except StopIteration:
                    self.finished[r] = True
                    continue
            while pending[r] and len(active[r]) < self.resident:
                active[r].append(pending[r].pop(self.rng.randrange(len(pending[r]))))      # any dispatch order
            g = self.rng.choice(active[r])
            try:
                res = next(g)
            except StopIteration:
                active[r].remove(g)
                res = None
            idle = idle + 1 if (res == "wait" and not self.net) else 0
            if idle > 100_000:
                raise Violation("deadlock: only waiting CTAs and nothing in flight")
        raise Violation("simulation did not finish")


def test_ll_protocol_is_safe_under_random_schedules_and_delivery_orders():
    for seed in range(60):
        rng = random.Random(1000 + seed)
        n = rng.choice([2, 3, 4, 8])
        T = rng.choice([1, 2, 3, 5, 8, 13])
        LlSim(n, tokens=T, exchanges=7, resident=T, seed=seed).run()


def test_ll_protocol_with_a_different_row_count_every_exchange():
    """Eager steps: T changes between exchanges of the same slot (a 13-row prefill step followed by 3-row decode steps ...);
    rows that an exchange does not use keep an old tag and are simply never polled."""
    for seed in range(40):
        rng = random.Random(7 + seed)
        n = rng.choice([2, 4, 8])
        Ts = [rng.choice([1, 3, 6, 13]) for _ in range(8)]
        LlSim(n, tokens=0, exchanges=8, resident=max(Ts), seed=seed, tokens_per_exchange=Ts).run()


def test_ll_protocol_needs_every_cta_resident():
    """The simulator has teeth, and documents why residency matters: with fewer resident CTAs than launched and CTAs dispatched
    in any order, the CTAs that wait for a peer's rows can occupy every slot while the CTAs that would push to that peer cannot
    start."""
    dead = 0
    for seed in range(40):
        try:
            LlSim(2, tokens=6, exchanges=2, resident=1, seed=seed).run(max_steps=600_000)
        except Violation as e:
            dead += "deadlock" in str(e)
    assert dead > 0


def test_ll_protocol_is_safe_even_with_one_receive_slot():
    """The kernel alternates two receive slots because its callers alternate two partial buffers anyway (o_proj / down_proj), but
    the protocol does not depend on it: a rank can only push exchange k+1 into a peer's line after it finished k, which needed
    every row that peer owns - rows the peer normalised AFTER consuming that very line; and an owner's broadcast of k+1 needs the
    k+1 pushes of every rank, i.e. every rank has finished k.  The simulator agrees (it flags any overwrite of an unconsumed line
    and any tag match on a payload of another exchange)."""
    for seed in range(80):
        LlSim(3, tokens=4, exchanges=6, resident=4, seed=seed, slots=1).run()
