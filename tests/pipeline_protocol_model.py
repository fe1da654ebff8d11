"""TEST INFRASTRUCTURE: an executable model of the synchronisation protocols of the fused-attention kernel (both variants,
artdeco_b200/csrc/attn_tc.cu) and the GEMM (artdeco_b200/csrc/gemm_tc.cu), explored under random interleavings on the CPU.

Why: the kernels are warp-specialised pipelines glued together by mbarriers whose waits see only the PARITY of a phase.
A protocol in which a barrier can complete two phases before a waiter looks deadlocks on hardware (an earlier version of the
attention kernel hung under CUDA-graph replay this way) and no amount of single-kernel testing reliably shows it.  The
model reproduces exactly that semantics:

  * ``Barrier``  arrival count, phase counter; ``wait(parity)`` passes iff the parity of the CURRENT (incomplete) phase
                 differs from the awaited one -- so a waiter that is two phases late blocks forever, as on the GPU;
  * TMA loads    complete asynchronously and out of order (an agent picks any in-flight load);
  * wgmma        each consumer warp's wgmma groups read shared memory asynchronously, in issue order, and
                 ``wgmma.wait_group N`` blocks until at most N of the warp's groups are still in flight;
  * every agent (producer warps, consumer warps) is a generator that blocks on barrier waits; a seeded random
    scheduler picks which runnable agent advances.

Besides deadlock the model checks the DATA hazards with explicit state for the Q buffer and the K / V / GEMM ring stages:
every read finds the load it expects, and no load overwrites a buffer before all eight consumer warps have read it (e.g.
"Q is not replaced while score products of the current item still read it").

The transcription follows the kernels line by line; the barrier names are the kernels' enum names.
"""
from __future__ import annotations

import random
from collections import deque


class Hazard(AssertionError):
    pass


class Barrier:
    def __init__(self, name, count):
        self.name, self.count, self.pending, self.phase = name, count, count, 0

    def arrive(self):
        self.pending -= 1
        if self.pending < 0:
            raise Hazard(f"{self.name}: more arrivals than its count in one phase")
        if self.pending == 0:
            self.phase += 1
            self.pending = self.count

    def passed(self, parity):          # mbarrier.try_wait.parity
        return (self.phase & 1) != (parity & 1)


class Machine:
    """Shared substrate: barriers, the in-order tensor pipe, the out-of-order TMA engine, a random scheduler."""

    def __init__(self, seed):
        self.rng = random.Random(seed)
        self.bars = {}
        self.pipes = {}           # per consumer warp: in-flight wgmma groups (fn), executed in issue order
        self.loads = []           # (fn, barrier name)
        self.agents = {}

    def bar(self, name, count=None):
        if name not in self.bars:
            self.bars[name] = Barrier(name, count)
        return self.bars[name]

    # --- helpers used by the agent generators ---
    def wait(self, name, parity):
        b = self.bars[name]
        return lambda: b.passed(parity)

    def inflight_at_most(self, warp, n):   # wgmma.wait_group n
        q = self.pipes.setdefault(warp, deque())
        return lambda: len(q) <= n

    def issue(self, warp, fn):               # wgmma.mma_async ... ; wgmma.commit_group
        self.pipes.setdefault(warp, deque()).append(fn)

    def run(self, max_steps=2_000_000):
        blocked = {n: None for n in self.agents}
        gens = dict(self.agents)
        done = set()
        for n, g in gens.items():
            blocked[n] = next(g, StopIteration)
        steps = 0
        while True:
            steps += 1
            if steps > max_steps:
                raise Hazard("no progress bound exceeded")
            choices = [("agent", n) for n in gens if n not in done and (blocked[n] is StopIteration or blocked[n]())]
            for w, q in self.pipes.items():
                if q:
                    choices.append(("pipe", w))
            for i in range(len(self.loads)):
                choices.append(("load", i))
            if not choices:
                if len(done) == len(gens):
                    return steps
                stuck = {n: getattr(blocked[n], "__doc__", None) or "?" for n in gens if n not in done}
                raise Hazard(f"DEADLOCK; blocked agents: {sorted(stuck)}; phases: " +
                             ", ".join(f"{b.name}={b.phase}/{b.pending}" for b in self.bars.values()))
            kind, which = self.rng.choice(choices)
            if kind == "pipe":
                self.pipes[which].popleft()()
            elif kind == "load":
                fn, barname = self.loads.pop(which)
                fn()
                self.bars[barname].arrive()
            else:
                n = which
                if blocked[n] is StopIteration:
                    done.add(n)
                    continue
                nxt = next(gens[n], StopIteration)
                blocked[n] = nxt
                if nxt is StopIteration:
                    done.add(n)


class Buffer:
    """A shared-memory buffer filled by TMA and read by every consumer warp.  ``tag`` names the load it holds; ``load``
    refuses to overwrite contents that some warp has not finished reading."""

    def __init__(self, name, readers=8):
        self.name, self.readers, self.tag, self.reads = name, readers, None, readers

    def load(self, tag):
        def f():
            if self.reads < self.readers:
                raise Hazard(f"{self.name} overwritten with load {tag} while {self.readers - self.reads} warps still "
                             f"had to read load {self.tag}")
            self.tag, self.reads = tag, 0
        return f

    def read(self, tag):
        if self.tag != tag:
            raise Hazard(f"{self.name}: a read expected load {tag}, found {self.tag}")

    def done(self, tag):            # this warp's last read of the contents
        self.read(tag)
        self.reads += 1


# =====================================================================================================================
# attn_fused_kernel<TILES> (artdeco_b200/csrc/attn_tc.cu): warp 8 loads Q and the K blocks of both passes, warp 9 the V^T
# blocks, warps 0..7 (two warpgroups) compute.  TILES = 1: one item per CTA; TILES = 2: persistent CTAs over n_items.
# =====================================================================================================================
def attention(nb, n_items, tiles, seed, kst, vst):
    M = Machine(seed)
    M.bar("QFULL", 1); M.bar("QEMPTY", 8)
    for s in range(kst):
        M.bar(f"KFULL{s}", 1); M.bar(f"KEMPTY{s}", 8)
    for s in range(vst):
        M.bar(f"VFULL{s}", 1); M.bar(f"VEMPTY{s}", 8)
    Q = Buffer("Q")
    K = [Buffer(f"K stage {s}") for s in range(kst)]
    V = [Buffer(f"V stage {s}") for s in range(vst)]

    def producer_qk():
        kc = 0
        for wi in range(n_items):
            yield M.wait("QEMPTY", (wi & 1) ^ 1)
            M.loads.append((Q.load(wi), "QFULL"))
            for _ in range(2 * nb):                          # pass 1 then pass 2
                s = kc % kst
                yield M.wait(f"KEMPTY{s}", ((kc // kst) & 1) ^ 1)
                M.loads.append((K[s].load(kc), f"KFULL{s}"))
                kc += 1

    def producer_v():
        vc = 0
        for _ in range(n_items):
            for _ in range(nb):
                s = vc % vst
                yield M.wait(f"VEMPTY{s}", ((vc // vst) & 1) ^ 1)
                M.loads.append((V[s].load(vc), f"VFULL{s}"))
                vc += 1

    def consumer(w):
        def score(ks, kc, wi, last_q):                      # wgmma S = Q_t K^T; commit; wait_group 0
            def f():
                (Q.done if last_q else Q.read)(wi)
                K[ks].read(kc)
            M.issue(w, f)
            yield M.inflight_at_most(w, 0)

        def g():
            kc = vc = 0
            for wi in range(n_items):
                yield M.wait("QFULL", wi & 1)
                for _ in range(nb):                          # pass 1
                    ks = kc % kst
                    yield M.wait(f"KFULL{ks}", (kc // kst) & 1)
                    for _ in range(tiles):
                        yield from score(ks, kc, wi, False)
                    K[ks].done(kc)
                    M.bars[f"KEMPTY{ks}"].arrive()
                    kc += 1
                for j in range(nb):                          # pass 2
                    ks, vs = kc % kst, vc % vst
                    yield M.wait(f"KFULL{ks}", (kc // kst) & 1)
                    yield M.wait(f"VFULL{vs}", (vc // vst) & 1)
                    for t in range(tiles):
                        last = t == tiles - 1 and j == nb - 1
                        yield from score(ks, kc, wi, last)
                        if last:
                            M.bars["QEMPTY"].arrive()
                        M.issue(w, (lambda vs_, vc_: lambda: V[vs_].read(vc_))(vs, vc))     # wgmma O += P V
                        yield M.inflight_at_most(w, 0)
                    K[ks].done(kc)
                    V[vs].done(vc)
                    M.bars[f"KEMPTY{ks}"].arrive()
                    M.bars[f"VEMPTY{vs}"].arrive()
                    kc += 1
                    vc += 1
        return g

    M.agents = {"tma_qk": producer_qk(), "tma_v": producer_v()}
    for w in range(8):
        M.agents[f"consumer{w}"] = consumer(w)()
    return M


def variant1(nb, seed, kst=3, vst=3):
    """One 128-query tile per CTA, one work item."""
    return attention(nb, 1, 1, seed, kst, vst)


def variant2(nb, n_items, seed, kst=3, vst=2):
    """Two query tiles per persistent CTA, n_items work items."""
    return attention(nb, n_items, 2, seed, kst, vst)


# =====================================================================================================================
# gemm_tc_kernel (artdeco_b200/csrc/gemm_tc.cu): one CTA per output tile; warp 8 fills the TMA ring, warps 0..7 (two
# warpgroups) keep one k-block of wgmma in flight and release a ring slot one k-block late; the last slot of a K-chunk is
# released after wait_group 0, before the partial sum is promoted.  n_tiles CTAs run side by side.
# =====================================================================================================================
def gemm(n_tiles, num_kb, seed, stages=3, kchunk=8):
    M = Machine(seed)

    def cta(c):
        for s in range(stages):
            M.bar(f"full{c}.{s}", 1); M.bar(f"empty{c}.{s}", 8)
        ring = [Buffer(f"CTA {c} stage {s}") for s in range(stages)]

        def producer():
            for kb in range(num_kb):
                s = kb % stages
                yield M.wait(f"empty{c}.{s}", ((kb // stages) & 1) ^ 1)
                M.loads.append((ring[s].load(kb), f"full{c}.{s}"))

        def consumer(w):
            me = (c, w)

            def g():
                for kb0 in range(0, num_kb, kchunk):
                    kb1 = min(kb0 + kchunk, num_kb)
                    for kb in range(kb0, kb1):
                        s = kb % stages
                        yield M.wait(f"full{c}.{s}", (kb // stages) & 1)
                        M.issue(me, (lambda s_, kb_: lambda: ring[s_].done(kb_))(s, kb))
                        yield M.inflight_at_most(me, 1)
                        if kb > kb0:
                            M.bars[f"empty{c}.{(kb - 1) % stages}"].arrive()
                    yield M.inflight_at_most(me, 0)
                    M.bars[f"empty{c}.{(kb1 - 1) % stages}"].arrive()
            return g

        M.agents[f"tma{c}"] = producer()
        for w in range(8):
            M.agents[f"consumer{c}.{w}"] = consumer(w)()

    for c in range(n_tiles):
        cta(c)
    return M
