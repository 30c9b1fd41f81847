#!/usr/bin/env python
"""Model check of the mbarrier protocol of the persistent convolution kernel (k_conv_wgmma in csrc/qnet.cu; k_wgrad_wgmma uses the
same ring with one tile per CTA).

The kernel's control flow is restated with the SAME index / parity expressions (stage = it % STAGES with a running round counter,
producer waits empty[s] with parity (round - 1) & 1, a consumer waits full[s] with a phase bit that flips when s wraps, and releases a
stage only after wgmma.wait_group 1 has reported the wgmmas that read it complete) and run under a randomised scheduler with
asynchronous completions (TMA transaction bytes and wgmma groups complete "later", in issue order per engine).  mbarriers are modelled
with their real semantics: a phase completes when the pending arrival count and the pending transaction bytes reach zero,
`try_wait.parity P` succeeds iff P differs from the parity of the phase in progress - so a waiter that is lapped would be fooled
exactly as on hardware.  Checked on every schedule:
  * no deadlock;
  * every wait passes in the phase it was meant for (no parity aliasing);
  * a ring stage is overwritten only after every consumer's wgmmas that read it completed, and is read only when completely filled
    with the k-step the consumer expects;
  * every tile is produced and consumed by every consumer warpgroup exactly once, in order.
Run: python tests/host/pipeline_protocol_check.py [schedules]
"""
import random
import sys


class Bar:
    def __init__(self, count):
        self.count, self.pending, self.tx, self.phase = count, count, 0, 0

    def _maybe_complete(self):
        if self.pending == 0 and self.tx == 0:
            self.phase += 1
            self.pending = self.count

    def arrive(self):
        assert self.pending > 0, "more arrivals than the barrier expects in one phase"
        self.pending -= 1
        self._maybe_complete()

    def expect_tx_arrive(self, nbytes):
        self.tx += nbytes
        self.arrive()

    def complete_tx(self, nbytes):
        self.tx -= nbytes
        assert self.tx >= 0
        self._maybe_complete()

    def ready(self, parity):
        return parity != (self.phase & 1)


def simulate(seed, stages, nk, ntiles, ncons=2, warps_per_cons=4, b_bytes=64):
    rng = random.Random(seed)
    full = [Bar(1) for _ in range(stages)]
    empty = [Bar(ncons * warps_per_cons) for _ in range(stages)]
    # ground truth bookkeeping
    stage_fill = [dict() for _ in range(stages)]  # (tile, kn) -> set of operands landed
    readers = [set() for _ in range(stages)]      # consumers whose wgmmas reading the stage have not completed
    consumed = [[] for _ in range(ncons)]
    reads = {}                                    # (stage, tile, k-step) -> consumers that read it
    deferred = []                                 # asynchronous completions: (engine, callable), executed in order per engine
    group_done = [dict() for _ in range(ncons)]   # consumer -> {issue index: completed}

    def producer():
        sn, rnd = 0, 0
        for t in range(ntiles):
            for kn in range(nk):
                if rnd > 0:
                    yield ("wait", empty[sn], (rnd - 1) & 1, rnd - 1, "producer empty[%d]" % sn)
                full[sn].expect_tx_arrive(2 * b_bytes)
                for op in ("A", "B"):
                    def land(s=sn, tt=t, kk=kn, o=op):
                        assert not readers[s], "stage %d (%s) overwritten before the wgmmas of %s completed" % (s, o, sorted(readers[s]))
                        for old in [key for key in stage_fill[s] if key != (tt, kk)]:
                            assert reads.get((s,) + old, 0) == ncons, "stage %d overwritten before every consumer read k-step %s" % (s, old)
                            del stage_fill[s][old]
                        stage_fill[s].setdefault((tt, kk), set()).add(o)
                        full[s].complete_tx(b_bytes)
                    defer("tma", land)
                yield ("step",)
                sn += 1
                if sn == stages:
                    sn, rnd = 0, rnd + 1

    def defer(engine, fn):
        deferred.append((engine, fn))

    def release(c, s):
        for _ in range(warps_per_cons):  # one arrival per consumer warp after its wgmma.wait_group
            empty[s].arrive()

    def consumer(c):
        s, ph, it = 0, 0, 0
        for i in range(ntiles):
            prev = None
            for kb in range(nk):
                yield ("wait", full[s], ph, it // stages, "consumer %d full[%d]" % (c, s))
                fill = stage_fill[s].get((i, kb))
                assert fill == {"A", "B"}, "consumer %d, tile %d k-step %d read stage %d holding %s" % (c, i, kb, s, stage_fill[s])
                readers[s].add(c)
                idx = it

                reads[(s, i, kb)] = reads.get((s, i, kb), 0) + 1

                def done(ss=s, n=idx):
                    readers[ss].discard(c)
                    group_done[c][n] = True
                defer("wgmma%d" % c, done)
                yield ("step",)
                # wgmma.wait_group 1: every group but the one just committed has completed
                if prev is not None:
                    yield ("until", lambda n=prev[1]: group_done[c].get(n, False), "consumer %d wait_group 1" % c)
                    release(c, prev[0])
                prev = (s, idx)
                it += 1
                s += 1
                if s == stages:
                    s, ph = 0, ph ^ 1
            yield ("until", lambda n=prev[1]: group_done[c].get(n, False), "consumer %d wait_group 0" % c)
            release(c, prev[0])
            consumed[c].append(i)

    agents = [producer()] + [consumer(c) for c in range(ncons)]
    state = [next(g) for g in agents]
    alive = [True] * len(agents)

    def runnable(st):
        if st[0] == "step":
            return True
        if st[0] == "wait":
            return st[1].ready(st[2])
        return st[1]()

    while any(alive) or deferred:
        choices = [("agent", k) for k, st in enumerate(state) if alive[k] and runnable(st)]
        engines = []
        for eng, _ in deferred:
            if eng not in engines:
                engines.append(eng)  # the oldest completion of every engine may happen now
        choices += [("engine", e) for e in engines]
        if not choices:
            blocked = [st[-1] for k, st in enumerate(state) if alive[k] and st[0] != "step"]
            raise AssertionError("deadlock; blocked: %s" % blocked)
        kind, which = rng.choice(choices)
        if kind == "engine":
            for j, (eng, fn) in enumerate(deferred):
                if eng == which:
                    deferred.pop(j)
                    fn()
                    break
            continue
        st = state[which]
        if st[0] == "wait":
            bar, intended = st[1], st[3]
            assert bar.phase == intended + 1, "%s passed in phase %d, meant for the completion of phase %d (parity aliasing)" % (st[4], bar.phase, intended)
        try:
            state[which] = next(agents[which])
        except StopIteration:
            alive[which] = False
    for c in range(ncons):
        assert consumed[c] == list(range(ntiles))
    assert all(not r for r in readers)
    assert all(v == ncons for v in reads.values()) and len(reads) == ntiles * nk
    return True


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 300
    cases = 0
    for stages in (2, 3, 4, 6, 8):
        for nk in (1, 2, 4, 9, 36):
            for ntiles in (1, 2, 3, 5, 8):
                for r in range(max(1, n // 100)):
                    simulate(hash((stages, nk, ntiles, r)) & 0xffffffff, stages, nk, ntiles)
                    cases += 1
    for r in range(n):
        rr = random.Random(r)
        simulate(r, rr.choice((2, 3, 4, 6, 8)), rr.choice((1, 4, 9, 18, 36)), rr.choice((1, 2, 4, 7, 9)), ncons=rr.choice((1, 2)))
        cases += 1
    print("pipeline protocol: %d randomised schedules, no deadlock, no aliasing, no hazard" % cases)


if __name__ == "__main__":
    main()
