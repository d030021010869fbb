"""Exhaustive interleaving check of the mbarrier protocol of the own attention forward kernel (csrc/attention_wgmma.cu,
`attn_fwd_kernel`).  mbarrier phase / parity mistakes are the classic way such a kernel hangs or reads a stale tile, and they are a
property of the SYNCHRONISATION SKELETON, which can be executed on a CPU: every role (the TMA-issuing thread and the two consumer
warpgroups) is transcribed as a straight program of `wait(barrier, parity)` / `arrive` / asynchronous TMA loads / tensor-core work,
with the parity expressions copied from the kernel, and a small explicit-state explorer runs every interleaving (including
arbitrary delays of the TMA engine).  The CTA barrier that ends a key block is modelled as a barrier every role arrives on and then
waits for.  Checked: no deadlock, every role finishes, every read sees the K / V block it expects, and no stage is overwritten by a
TMA load before its last reader is done.

mbarrier semantics used: a barrier counts arrivals of the current phase; when the count is reached the phase number advances.
`try_wait.parity p` succeeds iff the phase with parity p has completed, i.e. iff the parity of the CURRENT phase differs from p."""
import pytest


class Model:
    """roles: {name: [instr, ...]};  instr = ("wait", bar, parity) | ("arrive", bar) | ("tma", bar, fn) | ("mma", fn) | ("commit", bar) | ("do", fn)
    fn(data: dict) mutates a copy of the data state and asserts the hazards."""

    def __init__(self, roles, barriers, data):
        self.names = sorted(roles)
        self.roles = roles
        self.bar_names = sorted(barriers)
        self.counts = barriers
        self.data0 = data

    def initial(self):
        pcs = tuple(0 for _ in self.names)
        bars = tuple((0, self.counts[b]) for b in self.bar_names)          # (phase, pending arrivals)
        return pcs, bars, (), (), tuple(sorted(self.data0.items()))        # + tensor FIFO, TMA in flight, data

    def _arrive(self, bars, b):
        i = self.bar_names.index(b)
        phase, pend = bars[i]
        pend -= 1
        if pend == 0:
            phase, pend = phase + 1, self.counts[b]
        return bars[:i] + ((phase, pend),) + bars[i + 1:]

    def successors(self, st):
        pcs, bars, fifo, tma, data = st
        out = []
        for r, name in enumerate(self.names):
            prog = self.roles[name]
            if pcs[r] >= len(prog):
                continue
            ins = prog[pcs[r]]
            npcs = pcs[:r] + (pcs[r] + 1,) + pcs[r + 1:]
            if ins[0] == "wait":
                phase, _ = bars[self.bar_names.index(ins[1])]
                if (phase & 1) != ins[2]:
                    out.append((npcs, bars, fifo, tma, data))
            elif ins[0] == "arrive":
                out.append((npcs, self._arrive(bars, ins[1]), fifo, tma, data))
            elif ins[0] == "tma":
                d = dict(data)
                ins[2](d, "issue")
                out.append((npcs, bars, fifo, tma + ((ins[1], ins[2]),), tuple(sorted(d.items()))))
            elif ins[0] in ("mma", "commit"):
                out.append((npcs, bars, fifo + (ins,), tma, data))
            elif ins[0] == "do":
                d = dict(data)
                ins[1](d)
                out.append((npcs, bars, fifo, tma, tuple(sorted(d.items()))))
        if fifo:                                                            # the tensor pipe retires its oldest operation
            ins = fifo[0]
            if ins[0] == "mma":
                d = dict(data)
                ins[1](d)
                out.append((pcs, bars, fifo[1:], tma, tuple(sorted(d.items()))))
            else:
                out.append((pcs, self._arrive(bars, ins[1]), fifo[1:], tma, data))
        for k, (b, fn) in enumerate(tma):                                   # any in-flight TMA load lands
            d = dict(data)
            fn(d, "land")
            out.append((pcs, self._arrive(bars, b), fifo, tma[:k] + tma[k + 1:], tuple(sorted(d.items()))))
        return out

    def explore(self):
        start = self.initial()
        seen, stack = {start}, [start]
        while stack:
            st = stack.pop()
            nxt = self.successors(st)
            if not nxt:
                pcs = st[0]
                stuck = {n: self.roles[n][pcs[i]] for i, n in enumerate(self.names) if pcs[i] < len(self.roles[n])}
                assert not stuck and not st[2] and not st[3], f"deadlock: {stuck}"
            for t in nxt:
                if t not in seen:
                    seen.add(t)
                    stack.append(t)
        return len(seen)


def named(name, fn):
    fn.__name__ = name          # instructions are compared / hashed by identity; the name only helps error messages
    return fn


# ================================================================================================ forward
def forward_model(nblk, break_parity=False):
    """attn_fwd_kernel: thread 0 issues Q and the first two K/V blocks, then block i + 2 into stage i & 1 after the CTA barrier that
    ends block i; both warpgroups wait full[i & 1] with parity (i >> 1) & 1, read the stage, and join the CTA barrier."""
    data = {"Q": False}
    for s in range(2):
        data[f"KV{s}"], data[f"KV{s}_readers"] = -1, 0

    def tma_kv(s, i):
        def fn(d, what):
            if what == "issue":
                assert d[f"KV{s}_readers"] == 0, f"TMA overwrites stage {s} (block {d[f'KV{s}']}) while it is read, with block {i}"
                d[f"KV{s}"] = -1
            else:
                d[f"KV{s}"] = i
        return named(f"tma_kv{s}_{i}", fn)

    def tma_q(d, what):
        if what == "land":
            d["Q"] = True

    def read_begin(w, i):
        def fn(d):
            s = i & 1
            assert d["Q"], f"warpgroup {w} reads Q before it landed"
            assert d[f"KV{s}"] == i, f"warpgroup {w} block {i} reads stage {s} holding block {d[f'KV{s}']}"
            d[f"KV{s}_readers"] += 1
        return named(f"read_begin{w}_{i}", fn)

    def read_end(w, i):
        def fn(d):
            d[f"KV{i & 1}_readers"] -= 1
        return named(f"read_end{w}_{i}", fn)

    producer = [("tma", "q_full", named("tma_q", tma_q)), ("tma", "full0", tma_kv(0, 0))]
    if nblk > 1:
        producer += [("tma", "full1", tma_kv(1, 1))]
    for i in range(nblk):
        producer += [("arrive", "cta"), ("wait", "cta", i & 1)]
        if i + 2 < nblk:
            producer += [("tma", f"full{i & 1}", tma_kv(i & 1, i + 2))]
    roles = {"producer": producer}
    for w in range(2):
        prog = [("wait", "q_full", 0)]
        for i in range(nblk):
            parity = ((i >> 1) & 1) if not break_parity else 0
            prog += [("wait", f"full{i & 1}", parity), ("do", read_begin(w, i)), ("do", read_end(w, i)), ("arrive", "cta"),
                     ("wait", "cta", i & 1)]
        roles[f"warpgroup{w}"] = prog
    bars = {"q_full": 1, "full0": 1, "full1": 1, "cta": 3}           # the CTA barrier: thread 0's warpgroup and the two consumers
    return Model(roles, bars, data)


@pytest.mark.parametrize("nblk", [1, 2, 3, 4, 5, 6])
def test_forward_protocol(nblk):
    assert forward_model(nblk).explore() > nblk * 10


def test_forward_checker_catches_a_parity_bug():
    with pytest.raises(AssertionError):
        forward_model(3, break_parity=True).explore()
