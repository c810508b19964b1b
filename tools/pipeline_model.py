"""Protocol model of the warp-specialised kernels: attention pipelines and the CTA-pair GEMM (CPU, no GPU needed).

The fused attention kernels are mbarrier pipelines between three kinds of actors: one TMA-producer thread, one
tcgen05.mma-issuer thread and 4 or 8 softmax warps.  A wrong phase parity does not necessarily hang: an mbarrier
parity wait passes whenever the barrier is in the *other* phase, so being two phases off silently lets a buffer be
overwritten while it is still being read.  This module replays each kernel's wait / arrive / commit / load sequence
(transcribed from the .cu files, same variable names) under randomised asynchronous completion orders and checks

  * liveness  - every actor finishes (no deadlock),
  * ordering  - every consumer sees exactly the buffer version it expects (no premature pass),
  * exclusion - no buffer is overwritten (TMA load, MMA write, softmax write) while a read of it is outstanding.

The one-shot backward kernel is validated on hardware; it is modelled too, so the model itself is calibrated against a
protocol that is known to be right.  `tests/test_pipeline_model.py` runs all protocols over many schedules.

mbarrier semantics modelled: `phase` = number of completed phases; wait(parity) passes iff (phase & 1) != parity;
tcgen05.commit arrives once every MMA issued before it has completed (in-order queue); a TMA load arrives on its
barrier when its bytes have landed (each load completes independently, at a random later time).
"""
from __future__ import annotations

import random
from typing import Dict, List


class ProtocolError(AssertionError):
    pass


class Bar:
    def __init__(self, name: str, count: int):
        self.name, self.count, self.pending, self.phase = name, count, 0, 0

    def arrive(self):
        self.pending += 1
        if self.pending == self.count:
            self.pending, self.phase = 0, self.phase + 1

    def passed(self, parity: int) -> bool:
        return (self.phase & 1) != (parity & 1)


class Buf:
    """A shared-memory or TMEM buffer with versioned contents."""

    def __init__(self, name: str, warps: int):
        self.name, self.warps = name, warps
        self.version = 0            # completed writes
        self.write_pending = False  # async write (TMA / MMA) in flight
        self.async_reads = 0        # MMA reads in flight
        self.parts = 0              # warps that have written their slice of the next version
        self.sync_reads: Dict[int, int] = {}  # version -> warps that have read it

    def check_writable(self, who: str, need_all_warp_reads: bool = False):
        if self.write_pending:
            raise ProtocolError(f"{who}: {self.name} written while a previous write is still in flight")
        if self.async_reads:
            raise ProtocolError(f"{who}: {self.name} overwritten while {self.async_reads} MMA read(s) are outstanding")
        if need_all_warp_reads and self.version > 0 and self.sync_reads.get(self.version, 0) < self.warps:
            raise ProtocolError(f"{who}: {self.name} v{self.version} overwritten before all {self.warps} warps read it "
                                f"({self.sync_reads.get(self.version, 0)} did)")

    def check_readable(self, who: str, version: int):
        if self.write_pending or self.parts:
            raise ProtocolError(f"{who}: {self.name} read while a write is in flight")
        if self.version != version:
            raise ProtocolError(f"{who}: {self.name} has version {self.version}, expected {version}")


class Sim:
    def __init__(self, seed: int):
        self.rng = random.Random(seed)
        self.bars: Dict[str, Bar] = {}
        self.bufs: Dict[str, Buf] = {}
        self.threads: Dict[str, object] = {}
        self.blocked: Dict[str, tuple] = {}
        self.mma_queue: List = []   # in-order completion events of the tensor pipe
        self.tma_events: List = []  # independent completion events

    def bar(self, name, count):
        self.bars[name] = Bar(name, count)
        return self.bars[name]

    def buf(self, name, warps=1):
        self.bufs[name] = Buf(name, warps)
        return self.bufs[name]

    # ---- actions yielded by the actors ----
    def do(self, who, act):
        kind = act[0]
        if kind == "arrive":
            act[1].arrive()
        elif kind == "commit":  # arrives after every MMA issued so far has completed
            bar = act[1]
            self.mma_queue.append(lambda: bar.arrive())
        elif kind == "mma":     # ("mma", reads=[(buf, version)], write=(buf, need_all_warp_reads) | None)
            reads, write = act[1], act[2]
            for b, v in reads:
                b.check_readable(who, v)
                b.async_reads += 1
            if write is not None:
                wb, need = write
                wb.check_writable(who, need)
                wb.write_pending = True

            def done():
                for b, _ in reads:
                    b.async_reads -= 1
                if write is not None:
                    write[0].write_pending = False
                    write[0].version += 1
            self.mma_queue.append(done)
        elif kind == "tma":     # ("tma", buf, bar)
            b, bar = act[1], act[2]
            b.check_writable(who)
            b.write_pending = True

            def landed():
                b.write_pending = False
                b.version += 1
                bar.arrive()
            self.tma_events.append(landed)
        elif kind == "read":    # synchronous read by one softmax warp
            b, v = act[1], act[2]
            b.check_readable(who, v)
            b.sync_reads[v] = b.sync_reads.get(v, 0) + 1
        elif kind == "write_part":  # one softmax warp writes its rows of the next version
            b = act[1]
            if b.parts == 0:
                b.check_writable(who)
            elif b.async_reads or b.write_pending:
                raise ProtocolError(f"{who}: {b.name} written while in use")
            b.parts += 1
            if b.parts == b.warps:
                b.parts, b.version = 0, b.version + 1
        else:
            raise ValueError(kind)

    def run(self, max_steps: int = 2_000_000):
        live = dict(self.threads)
        for _ in range(max_steps):
            if not live and not self.mma_queue and not self.tma_events:
                return
            choices = []
            for name in live:
                w = self.blocked.get(name)
                if w is None or w[0].passed(w[1]):
                    choices.append(("t", name))
            if self.mma_queue:
                choices.append(("m", None))
            for k in range(len(self.tma_events)):
                choices.append(("x", k))
            if not choices:
                waits = {n: (w[0].name, w[1], w[0].phase) for n, w in self.blocked.items() if n in live}
                raise ProtocolError(f"deadlock: {waits}")
            kind, arg = self.rng.choice(choices)
            if kind == "m":
                self.mma_queue.pop(0)()
            elif kind == "x":
                self.tma_events.pop(arg)()
            else:
                self.blocked.pop(arg, None)
                try:
                    act = next(live[arg])
                except StopIteration:
                    del live[arg]
                    continue
                if act[0] == "wait":
                    if not act[1].passed(act[2]):
                        self.blocked[arg] = (act[1], act[2])
                else:
                    self.do(arg, act)
        raise ProtocolError("step limit reached")


# ---------------------------------------------------------------------------------------------------------------
# attention_bwd_sm100.cu (one-shot; validated on hardware) and attention_bwd_persist_sm100.cu
# ---------------------------------------------------------------------------------------------------------------
def model_bwd(seed: int, n_items: int, nt: int, ts_bufs: int, warps: int, kT: bool, persistent: bool, bug: str = ""):
    """n_items must be 1 for the one-shot kernel.  `bug` injects a known protocol fault (used by the tests to show
    that the checker is sensitive): "no_x_empty", "y_empty_parity", "no_e_empty", "no_ts_empty" (and "no_acc_empty" / "no_stat_empty", which the
    model shows to be harmless: the accumulation of the next item already waits for d_full, which every warp only
    signals after its epilogue -- acc_empty and tp_empty are belt-and-braces waits)."""
    s = Sim(seed)
    W = warps
    x_full, x_empty = s.bar("x_full", 1), s.bar("x_empty", 1)
    y_full = [s.bar(f"y_full{i}", 1) for i in range(2)]
    y_empty = [s.bar(f"y_empty{i}", 1) for i in range(2)]
    ts_full = [s.bar(f"ts_full{i}", 1) for i in range(2)]
    ts_empty = [s.bar(f"ts_empty{i}", W) for i in range(2)]
    tp_full, tp_empty = s.bar("tp_full", 1), s.bar("tp_empty", W)
    e_full, e_empty = s.bar("e_full", W), s.bar("e_empty", 1)
    d_full, d_empty = s.bar("d_full", W), s.bar("d_empty", 1)
    acc_full, acc_empty = s.bar("acc_full", 1), s.bar("acc_empty", W)
    # round 2, dK/dV role of the persistent kernel: the item's per-query statistics (lse2 | delta) are two 1-D bulk
    # copies into a 2-stage shared-memory buffer, requested together with the resident tiles
    stats = persistent and kT
    stat_full = [s.bar(f"stat_full{i}", 1) for i in range(2)]
    stat_empty = [s.bar(f"stat_empty{i}", W) for i in range(2)]
    STAT = [s.buf(f"stat{i}", W) for i in range(2)]
    X = s.buf("X")
    Y = [s.buf(f"Y{i}") for i in range(2)]
    Ts = [s.buf(f"Ts{i}", W) for i in range(2)]
    Tp = s.buf("Tp", W)
    E, D = s.buf("sE", W), s.buf("sD", W)
    ACC = s.buf("acc", W)
    T = n_items * nt

    def load_stats(i):
        if stats:
            sg = i & 1
            if i >= 2 and bug != "no_stat_empty":
                yield ("wait", stat_empty[sg], ((i >> 1) - 1) & 1)
            yield ("tma", STAT[sg], stat_full[sg])

    def producer():
        yield from load_stats(0)
        yield ("tma", X, x_full)
        for t in range(T):
            i, j = divmod(t, nt)
            st = t & 1
            if t >= 2:
                yield ("wait", y_empty[st], ((t >> 1) - (0 if bug == "y_empty_parity" else 1)) & 1)
            yield ("tma", Y[st], y_full[st])
            if persistent and j == nt - 1 and i + 1 < n_items:
                if bug != "no_x_empty":
                    yield ("wait", x_empty, i & 1)
                yield from load_stats(i + 1)
                yield ("tma", X, x_full)

    def mma():
        def prefetch_ts(t1):
            i1, j1 = divmod(t1, nt)
            s1, tb1 = t1 & 1, t1 % ts_bufs
            if j1 == 0:
                yield ("wait", x_full, i1 & 1)
            yield ("wait", y_full[s1], (t1 >> 1) & 1)
            if t1 >= ts_bufs and bug != "no_ts_empty":
                yield ("wait", ts_empty[tb1], (t1 // ts_bufs - 1) & 1)
            yield ("mma", [(X, i1 + 1), (Y[s1], (t1 >> 1) + 1)], (Ts[tb1], True))
            yield ("commit", ts_full[tb1])

        yield from prefetch_ts(0)
        for t in range(T):
            i, j = divmod(t, nt)
            st = t & 1
            last = j == nt - 1
            if t > 0:
                yield ("wait", tp_empty, (t - 1) & 1)
            yield ("mma", [(X, i + 1), (Y[st], (t >> 1) + 1)], (Tp, True))
            yield ("commit", tp_full)
            if persistent and last:
                yield ("commit", x_empty)
            if t + 1 < T and not (persistent and last):
                yield from prefetch_ts(t + 1)
            if persistent and j == 0 and i > 0 and bug != "no_acc_empty":
                yield ("wait", acc_empty, (i - 1) & 1)
            if kT:
                yield ("wait", e_full, t & 1)
                yield ("mma", [(E, t + 1), (Y[st], (t >> 1) + 1)], None)   # acc2 (same TMEM hazards as acc1)
                yield ("commit", e_empty)
            yield ("wait", d_full, t & 1)
            # the first accumulation of an item overwrites O: every warp must have read the previous item's O
            if j == 0:
                yield ("mma", [(D, t + 1), (Y[st], (t >> 1) + 1)], (ACC, True))
            else:
                yield ("mma", [(D, t + 1), (Y[st], (t >> 1) + 1)], None)
            yield ("commit", d_empty)
            yield ("commit", y_empty[st])
            if last:
                yield ("commit", acc_full)
                if persistent and t + 1 < T:
                    yield from prefetch_ts(t + 1)

    def softmax(w):
        for i in range(n_items):
            if stats:
                yield ("wait", stat_full[i & 1], (i >> 1) & 1)
            for j in range(nt):
                t = i * nt + j
                tb = t % ts_bufs
                yield ("wait", ts_full[tb], (t // ts_bufs) & 1)
                if stats:  # lse2 / delta of this tile's columns come out of the item's statistics stage
                    STAT[i & 1].check_readable(f"softmax{w}", (i >> 1) + 1)
                if kT and t > 0 and bug != "no_e_empty":
                    yield ("wait", e_empty, (t - 1) & 1)
                yield ("read", Ts[tb], t // ts_bufs + 1)
                if kT:
                    yield ("write_part", E)
                yield ("arrive", ts_empty[tb])
                if kT:
                    yield ("arrive", e_full)
                yield ("wait", tp_full, t & 1)
                if t > 0:
                    yield ("wait", d_empty, (t - 1) & 1)
                yield ("read", Tp, t + 1)
                yield ("write_part", D)
                yield ("arrive", tp_empty)
                yield ("arrive", d_full)
            if stats:
                yield ("read", STAT[i & 1], (i >> 1) + 1)
                yield ("arrive", stat_empty[i & 1])
            yield ("wait", acc_full, i & 1)
            yield ("read", ACC, i + 1)
            if persistent:
                yield ("arrive", acc_empty)

    s.threads["producer"] = producer()
    s.threads["mma"] = mma()
    for w in range(W):
        s.threads[f"softmax{w}"] = softmax(w)
    s.run()
    return s


# ---------------------------------------------------------------------------------------------------------------
# attention_persist_sm100.cu: persistent forward
# ---------------------------------------------------------------------------------------------------------------
def model_fwd_persist(seed: int, n_items: int, nkt: int, warps: int = 4, bug: str = ""):
    """Round-2 kernel: 4 softmax warps (row max, exp2, P ring, 1/sum into s_inv[item & 1]) and 4 separate epilogue
    warps (wait stat_full[item & 1] -> read s_inv -> wait acc_full -> read O -> arrive acc_empty).  The s_inv slot is a
    plain shared-memory hand-off between generic-proxy threads ordered ONLY by the stat_full mbarrier -- the pair
    compute-sanitizer racecheck reports.  bug="no_stat_full" drops that wait (the model must
    then see the epilogue read a stale / half-written slot); bug="stat_single" uses one slot instead of two."""
    s = Sim(seed)
    W = warps
    qk_full, qk_empty = s.bar("qk_full", 1), s.bar("qk_empty", 1)
    s_full, s_empty = s.bar("s_full", 1), s.bar("s_empty", W)
    acc_full, acc_empty = s.bar("acc_full", 1), s.bar("acc_empty", W)
    v_full = [s.bar(f"v_full{i}", 1) for i in range(2)]
    v_empty = [s.bar(f"v_empty{i}", 1) for i in range(2)]
    e_full = [s.bar(f"e_full{i}", W) for i in range(2)]
    e_empty = [s.bar(f"e_empty{i}", 1) for i in range(2)]
    stat_full = [s.bar(f"stat_full{i}", W) for i in range(2)]
    QK = s.buf("QK")
    V = [s.buf(f"V{i}") for i in range(2)]
    E = [s.buf(f"E{i}", W) for i in range(2)]
    S = s.buf("S", W)
    ACC = s.buf("O", W)
    SINV = [s.buf(f"s_inv{i}", W) for i in range(2)]
    slot = (lambda i: 0) if bug == "stat_single" else (lambda i: i & 1)

    def producer():
        def load_v(i, j):
            t = i * nkt + j
            st = t & 1
            if t >= 2:
                yield ("wait", v_empty[st], ((t >> 1) - 1) & 1)
            yield ("tma", V[st], v_full[st])

        yield ("tma", QK, qk_full)
        for i in range(n_items):
            first = min(nkt, 2)
            for j in range(first):
                yield from load_v(i, j)
            if i + 1 < n_items:
                yield ("wait", qk_empty, i & 1)
                yield ("tma", QK, qk_full)
            for j in range(first, nkt):
                yield from load_v(i, j)

    def mma():
        for i in range(n_items):
            yield ("wait", qk_full, i & 1)
            if i > 0:
                yield ("wait", s_empty, (i - 1) & 1)
            yield ("mma", [(QK, i + 1)], (S, True))
            yield ("commit", s_full)
            yield ("commit", qk_empty)
            if i > 0:
                yield ("wait", acc_empty, (i - 1) & 1)
            for j in range(nkt):
                t = i * nkt + j
                st = t & 1
                yield ("wait", v_full[st], (t >> 1) & 1)
                yield ("wait", e_full[st], (t >> 1) & 1)
                yield ("mma", [(E[st], (t >> 1) + 1), (V[st], (t >> 1) + 1)], (ACC, True) if j == 0 else None)
                yield ("commit", e_empty[st])
                yield ("commit", v_empty[st])
            yield ("commit", acc_full)

    def softmax(w):
        for i in range(n_items):
            yield ("wait", s_full, i & 1)
            yield ("read", S, i + 1)  # pass 1 (row max) and pass 2 read the same version
            for j in range(nkt):
                t = i * nkt + j
                eb = t & 1
                if t >= 2:
                    yield ("wait", e_empty[eb], ((t >> 1) - 1) & 1)
                S.check_readable(f"softmax{w}", i + 1)
                yield ("write_part", E[eb])
                yield ("arrive", e_full[eb])
            # 1 / row sum for the epilogue warps: every epilogue warp must have read the slot's previous contents
            sl = SINV[slot(i)]
            if sl.parts == 0 and sl.version > 0 and sl.sync_reads.get(sl.version, 0) < W:
                raise ProtocolError(f"softmax{w}: {sl.name} v{sl.version} overwritten before every epilogue warp read it")
            yield ("write_part", sl)
            yield ("arrive", s_empty)
            yield ("arrive", stat_full[slot(i)])

    def epilogue(w):
        for i in range(n_items):
            k = i if bug == "stat_single" else (i >> 1)
            if bug != "no_stat_full":
                yield ("wait", stat_full[slot(i)], k & 1)
            yield ("read", SINV[slot(i)], k + 1)
            yield ("wait", acc_full, i & 1)
            yield ("read", ACC, i + 1)
            yield ("arrive", acc_empty)

    s.threads["producer"] = producer()
    s.threads["mma"] = mma()
    for w in range(W):
        s.threads[f"softmax{w}"] = softmax(w)
        s.threads[f"epilogue{w}"] = epilogue(w)
    s.run()
    return s


# ---------------------------------------------------------------------------------------------------------------
# attention_bwd_sm100.cu: attn_fwd_long_sm100_kernel (two passes over the key tiles)
# ---------------------------------------------------------------------------------------------------------------
def model_fwd_long(seed: int, nt: int, warps: int = 4):
    s = Sim(seed)
    W = warps
    x_full = s.bar("x_full", 1)
    y_full = [s.bar(f"y_full{i}", 1) for i in range(2)]
    y_empty = [s.bar(f"y_empty{i}", 1) for i in range(2)]
    ts_full = [s.bar(f"ts_full{i}", 1) for i in range(2)]
    ts_empty = [s.bar(f"ts_empty{i}", W) for i in range(2)]
    e_full, e_empty = s.bar("e_full", W), s.bar("e_empty", 1)
    acc_done = s.bar("acc_done", 1)
    Q = s.buf("Q")
    Y = [s.buf(f"Y{i}") for i in range(2)]
    Ts = [s.buf(f"Ts{i}", W) for i in range(2)]
    E = s.buf("sE", W)
    nl = 2 * nt

    def producer():
        yield ("tma", Q, x_full)
        for l in range(nl):
            st = l & 1
            if l >= 2:
                yield ("wait", y_empty[st], ((l >> 1) - 1) & 1)
            yield ("tma", Y[st], y_full[st])

    def mma():
        yield ("wait", x_full, 0)
        for l in range(nl):
            st = l & 1
            if l == 0:
                yield ("wait", y_full[0], 0)
                yield ("mma", [(Q, 1), (Y[0], 1)], (Ts[0], True))
                yield ("commit", ts_full[0])
            if l < nt:
                yield ("commit", y_empty[st])
            if l + 1 < nl:
                l1 = l + 1
                s1 = l1 & 1
                yield ("wait", y_full[s1], (l1 >> 1) & 1)
                if l1 >= 2:
                    yield ("wait", ts_empty[s1], ((l1 >> 1) - 1) & 1)
                yield ("mma", [(Q, 1), (Y[s1], (l1 >> 1) + 1)], (Ts[s1], True))
                yield ("commit", ts_full[s1])
            if l >= nt:
                i = l - nt
                yield ("wait", e_full, i & 1)
                yield ("mma", [(E, i + 1), (Y[st], (l >> 1) + 1)], None)
                yield ("commit", e_empty)
                yield ("commit", y_empty[st])
        yield ("commit", acc_done)

    def softmax(w):
        for l in range(nt):
            yield ("wait", ts_full[l & 1], (l >> 1) & 1)
            yield ("read", Ts[l & 1], (l >> 1) + 1)
            yield ("arrive", ts_empty[l & 1])
        for l in range(nt, nl):
            i = l - nt
            yield ("wait", ts_full[l & 1], (l >> 1) & 1)
            if i > 0:
                yield ("wait", e_empty, (i - 1) & 1)
            yield ("read", Ts[l & 1], (l >> 1) + 1)
            yield ("write_part", E)
            yield ("arrive", ts_empty[l & 1])
            yield ("arrive", e_full)
        yield ("wait", acc_done, 0)

    s.threads["producer"] = producer()
    s.threads["mma"] = mma()
    for w in range(W):
        s.threads[f"softmax{w}"] = softmax(w)
    s.run()
    return s



# ---------------------------------------------------------------------------------------------------------------
# gemm_sm100.cu: CTA-pair tcgen05 GEMM with cluster-launch-control (CLC) work stealing
# ---------------------------------------------------------------------------------------------------------------
class TxBar(Bar):
    """mbarrier with a transaction count: the phase completes when all arrivals are in AND the tx-count is zero
    (complete_tx may land before the matching expect_tx: the count is transiently negative, which is legal)."""

    def __init__(self, name: str, count: int):
        super().__init__(name, count)
        self.tx = 0

    def _check(self):
        if self.pending == self.count and self.tx == 0:
            self.pending, self.phase = 0, self.phase + 1

    def arrive(self):
        self.pending += 1
        if self.pending > self.count:
            raise ProtocolError(f"{self.name}: more arrivals than the barrier expects in one phase")
        self._check()

    def expect_tx(self, n: int):
        self.tx += n
        self.arrive()

    def complete_tx(self, n: int):
        self.tx -= n
        self._check()


def model_gemm(seed: int, tiles: int, clusters: int = 2, num_kb: int = 3, stages: int = 3, clc_stages: int = 2,
               use_clc: bool = True, epi_warps: int = 8, epi_delay: int = 0, bug: str = ""):
    """`clusters` resident CTA pairs work through `tiles` output tiles.  Per pair: two TMA producers (one per CTA, both
    signalling the LEADER's full barrier, armed by the leader alone for the bytes of both), one MMA issuer (leader;
    its commits are multicast to both CTAs), one CLC scheduler (leader; responses multicast to both CTAs, 20
    consumers per response), 2 x `epi_warps` epilogue warps draining a double-buffered TMEM accumulator.

    Checked: liveness; every MMA reads the k-block it expects in BOTH CTAs' stages; every epilogue warp reads the
    accumulator of the tile it believes it is working on; nothing is overwritten while in use; all consumers of a pair
    walk the same tile sequence; every tile is computed exactly once.  bug = "no_empty" | "no_tmem_empty" |
    "no_clc_empty" | "peer_arms_too" (sensitivity of the checker).  epi_delay = idle scheduling slots an epilogue warp
    spends between learning that its accumulator is complete and reading it (real epilogues are slow; a uniformly random
    scheduler would otherwise almost never let the MMA issuer get two tiles ahead of them)."""
    s = Sim(seed)
    S_BYTES = 1  # bytes of one CTA's stage, in arbitrary units
    state = {"next": clusters}  # tiles 0 .. clusters-1 are the resident clusters' own; the rest are cancelled in order
    done_tiles: Dict[int, int] = {}
    n_consumers = 2 + 1 + 1 + 2 * epi_warps  # producers, MMA, scheduler, epilogue warps (= 20 in the kernel)

    def add_tag(buf):
        buf.tag = None
        return buf

    def build(cl):
        pre = f"c{cl}."
        full = [TxBar(pre + f"full{i}", 1) for i in range(stages)]
        empty = [[s.bar(pre + f"empty{c}_{i}", 1) for i in range(stages)] for c in range(2)]
        tmem_full = [[s.bar(pre + f"tmem_full{c}_{i}", 1) for i in range(2)] for c in range(2)]
        tmem_empty = [s.bar(pre + f"tmem_empty{i}", 2 * epi_warps) for i in range(2)]
        clc_full = [[TxBar(pre + f"clc_full{c}_{i}", 1) for i in range(clc_stages)] for c in range(2)]
        clc_empty = [s.bar(pre + f"clc_empty{i}", n_consumers) for i in range(clc_stages)]
        smem = [[add_tag(s.buf(pre + f"smem{c}_{i}")) for i in range(stages)] for c in range(2)]
        acc = [add_tag(s.buf(pre + f"acc{i}", 2 * epi_warps)) for i in range(2)]
        resp = [[add_tag(s.buf(pre + f"resp{c}_{i}", 1)) for i in range(clc_stages)] for c in range(2)]
        for row in clc_full:
            for b in row:
                s.bars[b.name] = b
        for b in full:
            s.bars[b.name] = b

        class TileIter:
            def __init__(self):
                self.tile, self.stage, self.phase, self.n = cl, 0, 0, 0

        def tile_next(it, c, who, arrive=True, full=clc_full, empty_=clc_empty, resp=resp, cl=cl):
            """generator: the consumer side of one CLC response; sets it.tile / returns validity in it.more"""
            if not use_clc:
                it.tile += clusters
                it.more = it.tile < tiles
                return
            yield ("wait", full[c][it.stage], it.phase)
            r = resp[c][it.stage]
            if r.write_pending:
                raise ProtocolError(f"{who}: CLC response slot {r.name} read while the hardware is writing it")
            if r.version != it.n // clc_stages + 1:  # it.n-th response overall = (it.n // stages + 1)-th use of this slot
                raise ProtocolError(f"{who}: CLC response slot {r.name} holds its response #{r.version}, expected "
                                    f"#{it.n // clc_stages + 1} (overwritten before it was consumed, or read early)")
            val = r.tag
            r.sync_reads[r.version] = r.sync_reads.get(r.version, 0) + 1
            if arrive:
                yield ("arrive", empty_[it.stage])
            it.stage = 0 if it.stage + 1 == clc_stages else it.stage + 1
            it.phase ^= 1 if it.stage == 0 else 0
            it.n += 1
            it.more = val is not None
            if it.more:
                it.tile = val

        def producer(c, full=full, empty=empty, smem=smem, pre=pre):
            who = pre + f"producer{c}"
            it = TileIter()
            stage = phase = 0
            it.more = it.tile < tiles
            while it.more:
                for kb in range(num_kb):
                    if bug != "no_empty":
                        yield ("wait", empty[c][stage], phase ^ 1)
                    yield ("gemm_tma", smem[c][stage], full[stage], S_BYTES, (it.tile, kb), who)
                    if c == 0 or bug == "peer_arms_too":
                        yield ("expect_tx", full[stage], 2 * S_BYTES)
                    stage = 0 if stage + 1 == stages else stage + 1
                    phase ^= 1 if stage == 0 else 0
                yield from tile_next(it, c, who)

        def mma(full=full, empty=empty, smem=smem, acc=acc, tmem_full=tmem_full, tmem_empty=tmem_empty, pre=pre):
            who = pre + "mma"
            it = TileIter()
            stage = phase = 0
            n = 0
            it.more = it.tile < tiles
            while it.more:
                a, aphase = n & 1, (n >> 1) & 1
                if bug != "no_tmem_empty":
                    yield ("wait", tmem_empty[a], aphase ^ 1)
                for kb in range(num_kb):
                    yield ("wait", full[stage], phase)
                    yield ("gemm_mma", [smem[0][stage], smem[1][stage]], (it.tile, kb), acc[a], kb == 0, who)
                    yield ("commit2", [empty[0][stage], empty[1][stage]])
                    if kb == num_kb - 1:
                        yield ("commit2", [tmem_full[0][a], tmem_full[1][a]])
                    stage = 0 if stage + 1 == stages else stage + 1
                    phase ^= 1 if stage == 0 else 0
                n += 1
                yield from tile_next(it, 0, who)
            if n > 0:  # drain: every epilogue warp of both CTAs released the last accumulators
                last = n - 1
                yield ("wait", tmem_empty[last & 1], (last >> 1) & 1)
                if n > 1:
                    prev = n - 2
                    yield ("wait", tmem_empty[prev & 1], (prev >> 1) & 1)

        def scheduler(clc_full=clc_full, clc_empty=clc_empty, resp=resp, pre=pre):
            who = pre + "scheduler"
            it = TileIter()
            stage = phase = 0
            it.more = it.tile < tiles
            while it.more:
                if bug != "no_clc_empty":
                    yield ("wait", clc_empty[stage], phase ^ 1)
                yield ("expect_tx", clc_full[0][stage], 16)
                yield ("expect_tx", clc_full[1][stage], 16)
                yield ("clc", [resp[0][stage], resp[1][stage]], [clc_full[0][stage], clc_full[1][stage]], who)
                stage = 0 if stage + 1 == clc_stages else stage + 1
                phase ^= 1 if stage == 0 else 0
                yield from tile_next(it, 0, who)

        def epilogue(c, w, acc=acc, tmem_full=tmem_full, tmem_empty=tmem_empty, pre=pre):
            who = pre + f"epi{c}_{w}"
            it = TileIter()
            n = 0
            it.more = it.tile < tiles
            while it.more:
                a, aphase = n & 1, (n >> 1) & 1
                yield ("wait", tmem_full[c][a], aphase)
                for _ in range(s.rng.randrange(epi_delay + 1)):
                    yield ("nop",)
                yield ("gemm_acc_read", acc[a], it.tile, who)
                yield ("arrive", tmem_empty[a])
                done_tiles[(it.tile, c, w)] = done_tiles.get((it.tile, c, w), 0) + 1
                n += 1
                yield from tile_next(it, c, who)

        s.threads[pre + "producer0"] = producer(0)
        s.threads[pre + "producer1"] = producer(1)
        s.threads[pre + "mma"] = mma()
        if use_clc:
            s.threads[pre + "scheduler"] = scheduler()
        for c in range(2):
            for w in range(epi_warps):
                s.threads[pre + f"epi{c}_{w}"] = epilogue(c, w)

    for cl_ in range(clusters):
        build(cl_)

    base_do = s.do

    def do(who, act):
        kind = act[0]
        if kind == "nop":
            pass
        elif kind == "expect_tx":
            act[1].expect_tx(act[2])
        elif kind == "gemm_tma":  # one CTA's half of a k-block into its own stage; bytes counted on the leader's barrier
            _, b, bar, nbytes, tag, _who = act
            b.check_writable(who)
            b.write_pending = True

            def landed():
                b.write_pending = False
                b.version += 1
                b.tag = tag
                bar.complete_tx(nbytes)
            s.tma_events.append(landed)
        elif kind == "gemm_mma":  # reads both CTAs' stage, accumulates into (or overwrites) the TMEM buffer
            _, bufs, tag, accb, first, _who = act
            for b in bufs:
                if b.write_pending:
                    raise ProtocolError(f"{who}: {b.name} read while a TMA write is in flight")
                if b.tag != tag:
                    raise ProtocolError(f"{who}: {b.name} holds k-block {b.tag}, expected {tag}")
                b.async_reads += 1
            if first:
                if accb.async_reads:
                    raise ProtocolError(f"{who}: {accb.name} overwritten while MMAs still read it")
                if accb.version > 0 and accb.sync_reads.get(accb.version, 0) < accb.warps:
                    raise ProtocolError(f"{who}: {accb.name} (tile {accb.tag}) overwritten before all {accb.warps} "
                                        f"epilogue warps read it ({accb.sync_reads.get(accb.version, 0)} did)")
                accb.version += 1
                accb.tag = tag[0]
            elif accb.tag != tag[0]:
                raise ProtocolError(f"{who}: accumulating tile {tag[0]} into {accb.name} which holds tile {accb.tag}")
            accb.write_pending = True

            def done():
                for b in bufs:
                    b.async_reads -= 1
                accb.write_pending = False
            s.mma_queue.append(done)
        elif kind == "commit2":  # multicast tcgen05.commit: arrives on both CTAs' barriers once prior MMAs completed
            bars = act[1]
            s.mma_queue.append(lambda: [b.arrive() for b in bars])
        elif kind == "gemm_acc_read":
            _, accb, tile, _who = act
            if accb.write_pending:
                raise ProtocolError(f"{who}: {accb.name} read while MMAs are still writing it")
            if accb.tag != tile:
                raise ProtocolError(f"{who}: reads {accb.name} for tile {tile} but it holds tile {accb.tag}")
            accb.sync_reads[accb.version] = accb.sync_reads.get(accb.version, 0) + 1
        elif kind == "clc":  # clusterlaunchcontrol.try_cancel, response multicast to both CTAs
            _, resps, bars, _who = act
            for r in resps:
                if r.write_pending:
                    raise ProtocolError(f"{who}: CLC request into {r.name} while the previous one is in flight")
                r.write_pending = True

            def answered():
                t = state["next"] if state["next"] < tiles else None
                if t is not None:
                    state["next"] += 1
                for r, b in zip(resps, bars):
                    r.write_pending = False
                    r.version += 1
                    r.tag = t
                    b.complete_tx(16)
            s.tma_events.append(answered)
        else:
            base_do(who, act)

    s.do = do
    s.run()
    # every tile exactly once, by every epilogue warp of both CTAs of exactly one pair
    for t in range(tiles):
        for c in range(2):
            for w in range(epi_warps):
                if done_tiles.get((t, c, w), 0) != 1:
                    raise ProtocolError(f"tile {t} processed {done_tiles.get((t, c, w), 0)} times by epilogue warp {c}/{w}")
    return s


# ---------------------------------------------------------------------------------------------------------------
# gemm_sm90.cu with kClusterM = 2: CTA pairs along M, B tile multicast, static persistent schedule
# ---------------------------------------------------------------------------------------------------------------
class _CtaBar(TxBar):
    """An mbarrier in one CTA's shared memory: arriving on it or completing bytes on it after that CTA exited is a
    fault (the smem may already belong to another CTA)."""

    def __init__(self, name: str, count: int, cta: dict):
        super().__init__(name, count)
        self.cta = cta

    def arrive(self):
        if self.cta["exited"]:
            raise ProtocolError(f"{self.name}: arrival after its CTA exited")
        super().arrive()

    def complete_tx(self, n: int):
        if self.cta["exited"]:
            raise ProtocolError(f"{self.name}: bytes landed after its CTA exited")
        super().complete_tx(n)


def model_gemm_sm90_pair(seed: int, m_tiles: int, n_tiles: int, batch: int = 1, clusters: int = 2, num_kb: int = 3,
                         stages: int = 3, bug: str = ""):
    """`clusters` resident 2-CTA clusters walk units u = cluster, cluster + clusters, ... of m_units x n_tiles x batch
    (m_units = ceil(m_tiles / 2)); CTA c of a cluster computes m-tile 2 mu + c (with odd m_tiles the last pair's second
    CTA computes a tile below the matrix and still runs the whole protocol).  Per CTA: one TMA producer (expect_tx of
    the whole stage on its own full barrier, its A tile to itself, its B half multicast to both CTAs, each copy
    completing bytes on the receiving CTA's full barrier) and two consumer warpgroups (wgmma reads of A and both B
    halves, one k-block in flight, each of their 4 warps releasing the stage on both CTAs' empty barriers of 16
    arrivals); every thread meets the final cluster sync before its CTA exits.

    Checked: liveness; every wgmma reads the k-block it expects in all three parts of its stage; no part of a stage is
    overwritten while a read is outstanding; no barrier of an exited CTA is touched; every real tile is computed once
    by each warpgroup.  bug = "local_only" (consumers release only their own CTA's stage, barriers counting 8) |
    "no_final_sync" | "wait_peer_full" (a producer waits for the peer's full barrier instead of its own empty one)."""
    s = Sim(seed)
    A_BYTES, B_HALF = 2, 1  # bytes per stage part, in arbitrary units
    m_units = (m_tiles + 1) // 2
    per_batch = m_units * n_tiles
    total = per_batch * batch
    done: Dict[tuple, int] = {}
    ctas = []

    def tagged(name):
        b = s.buf(name)
        b.tag = None
        return b

    def build(cl):
        pre = f"c{cl}."
        cta = [{"exited": False, "live": 3} for _ in range(2)]  # producer + 2 consumer warpgroups
        ctas.extend(cta)
        empty_count = 4 * 2 * (1 if bug == "local_only" else 2)
        full = [[_CtaBar(pre + f"full{c}_{i}", 1, cta[c]) for i in range(stages)] for c in range(2)]
        empty = [[_CtaBar(pre + f"empty{c}_{i}", empty_count, cta[c]) for i in range(stages)] for c in range(2)]
        for row in full + empty:
            for b in row:
                s.bars[b.name] = b
        sa = [[tagged(pre + f"a{c}_{i}") for i in range(stages)] for c in range(2)]
        sb = [[[tagged(pre + f"b{c}_{i}_h{h}") for h in range(2)] for i in range(stages)] for c in range(2)]
        exit_sync = s.bar(pre + "cluster_sync", 6)
        units = list(range(cl, total, clusters))

        def teardown(c):
            if bug != "no_final_sync":
                yield ("arrive", exit_sync)
                yield ("wait", exit_sync, 0)
            yield ("exit", cta[c])

        def producer(c):
            stage = phase = 0
            for u in units:
                for kb in range(num_kb):
                    if bug == "wait_peer_full":
                        yield ("wait", full[1 - c][stage], phase ^ 1)
                    else:
                        yield ("wait", empty[c][stage], phase ^ 1)
                    yield ("expect_tx", full[c][stage], A_BYTES + 2 * B_HALF)
                    yield ("load", [(sa[c][stage], full[c][stage])], A_BYTES, (u, kb))
                    yield ("load", [(sb[d][stage][c], full[d][stage]) for d in range(2)], B_HALF, (u, kb))
                    stage = 0 if stage + 1 == stages else stage + 1
                    phase ^= 1 if stage == 0 else 0
            yield from teardown(c)

        def release(c, st):
            for _warp in range(4):
                for d in ([c] if bug == "local_only" else [0, 1]):
                    yield ("arrive", empty[d][st])

        def consumer(c, w):
            stage = phase = 0
            groups: List[list] = []  # committed wgmma groups not yet retired
            for u in units:
                b, r = divmod(u, per_batch)
                mu, nt = divmod(r, n_tiles)
                prev = 0
                for kb in range(num_kb):
                    yield ("wait", full[c][stage], phase)
                    yield ("wgmma", [sa[c][stage], sb[c][stage][0], sb[c][stage][1]], (u, kb), groups)
                    if kb > 0:
                        yield ("wgmma_wait", groups, 1)
                        yield from release(c, prev)
                    prev = stage
                    stage = 0 if stage + 1 == stages else stage + 1
                    phase ^= 1 if stage == 0 else 0
                yield ("wgmma_wait", groups, 0)
                yield from release(c, prev)
                key = (b, 2 * mu + c, nt, w)
                done[key] = done.get(key, 0) + 1
            yield from teardown(c)

        for c in range(2):
            s.threads[pre + f"producer{c}"] = producer(c)
            for w in range(2):
                s.threads[pre + f"wg{c}_{w}"] = consumer(c, w)

    for cl_ in range(clusters):
        build(cl_)

    base_do = s.do

    def do(who, act):
        kind = act[0]
        if kind == "expect_tx":
            act[1].expect_tx(act[2])
        elif kind == "load":  # one TMA box, landing (independently) in each destination CTA
            _, dests, nbytes, tag = act
            for b, _bar in dests:
                b.check_writable(who)
                b.write_pending = True
            for b, bar in dests:
                def landed(b=b, bar=bar):
                    b.write_pending = False
                    b.version += 1
                    b.tag = tag
                    bar.complete_tx(nbytes)
                s.tma_events.append(landed)
        elif kind == "wgmma":
            _, bufs, tag, groups = act
            for b in bufs:
                if b.write_pending:
                    raise ProtocolError(f"{who}: {b.name} read while a TMA write is in flight")
                if b.tag != tag:
                    raise ProtocolError(f"{who}: {b.name} holds k-block {b.tag}, expected {tag}")
                b.async_reads += 1
            groups.append(bufs)
        elif kind == "wgmma_wait":  # wgmma.wait_group N: all but the newest N groups have retired
            _, groups, n = act
            while len(groups) > n:
                for b in groups.pop(0):
                    b.async_reads -= 1
        elif kind == "exit":
            act[1]["live"] -= 1
            if act[1]["live"] == 0:
                act[1]["exited"] = True
        else:
            base_do(who, act)

    s.do = do
    s.run()
    if not all(c["exited"] for c in ctas):
        raise ProtocolError("a CTA never exited")
    for b in range(batch):
        for mt in range(m_tiles):
            for nt in range(n_tiles):
                for w in range(2):
                    if done.get((b, mt, nt, w), 0) != 1:
                        raise ProtocolError(f"tile {(b, mt, nt)} computed {done.get((b, mt, nt, w), 0)} times by "
                                            f"warpgroup {w}")
    return s


if __name__ == "__main__":
    for seed in range(200):
        model_bwd(seed, 1, 4, 2, 4, True, False)
        model_bwd(seed, 1, 4, 1, 4, True, False)
        model_bwd(seed, 1, 4, 2, 4, False, False)
        model_bwd(seed, 3, 4, 2, 8, True, True)
        model_bwd(seed, 3, 3, 2, 8, False, True)
        model_fwd_persist(seed, 3, 4)  # softmax + separate epilogue warps (round-2 kernel)
        model_fwd_long(seed, 9)
        model_gemm(seed, 9, clusters=2, epi_warps=2)
        model_gemm_sm90_pair(seed, 5, 3, batch=2, clusters=3)
    print("all protocols passed 200 schedules each")
