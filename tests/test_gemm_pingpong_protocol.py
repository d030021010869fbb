"""Exhaustive interleaving check of the synchronisation protocol of the ping-pong GEMM kernel (csrc/gemm_wgmma.cu,
`gemm_pingpong_kernel`), in the manner of `test_attention_protocol_model.py`.  The three roles - the TMA-issuing producer thread and the
two consumer warpgroups - are transcribed as straight programs of barrier waits / arrivals, asynchronous TMA loads, operand reads and
epilogue stores, with the ring positions and parity expressions of the kernel; a small explicit-state explorer runs every interleaving,
including any delay of a TMA load and any completion order of the bulk stores.  Checked:

* no deadlock: every role finishes;
* every operand read sees the k-block of the unit it expects (a unit's first stage is ring position i * num_k);
* no TMA load overwrites a stage before its reader released it;
* the order barrier serialises the mainloops: unit i starts issuing only after unit i - 1 issued its last k-block;
* no staging buffer is rewritten while a TMA store still reads it (`cp.async.bulk.wait_group.read 1` before each sub-tile).

The checker is shown to catch a missing order-barrier arrive, a wrong first-stage offset, a wrong order-barrier parity, a wrong
empty-barrier parity and a staging wait that leaves two stores in flight.

mbarrier semantics used: a barrier counts arrivals of the current phase; when the count is reached the phase number advances.
`try_wait.parity p` succeeds iff the phase with parity p has completed, i.e. iff the parity of the CURRENT phase differs from p."""
import pytest

NSUB = 4            # 64 x 64 output sub-tiles per 128 x 128 unit
NBUF = 2            # staging buffers per consumer warpgroup


class Model:
    """roles: {name: [instr, ...]}; instr = ("wait", bar, parity) | ("arrive", bar) | ("tma", bar, fn) | ("do", fn)
    | ("store", w, buf) | ("wait_read", w, n) | ("check_buf", w, buf).  fn(data) mutates a copy of the data state and asserts the
    hazards; a TMA fn is called with "issue" and "land"."""

    def __init__(self, roles, barriers, data):
        self.names = sorted(roles)
        self.roles = roles
        self.bar_names = sorted(barriers)
        self.counts = barriers
        self.data0 = data

    def initial(self):
        pcs = tuple(0 for _ in self.names)
        bars = tuple((0, self.counts[b]) for b in self.bar_names)            # (phase, pending arrivals)
        stores = ((0, ()), (0, ()))           # per warpgroup: (bulk groups committed, in-flight groups as (commit index, buffer))
        return pcs, bars, (), stores, tuple(sorted(self.data0.items()))

    def _arrive(self, bars, b):
        i = self.bar_names.index(b)
        phase, pend = bars[i]
        pend -= 1
        if pend == 0:
            phase, pend = phase + 1, self.counts[b]
        return bars[:i] + ((phase, pend),) + bars[i + 1:]

    def successors(self, st):
        pcs, bars, tma, stores, data = st
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
                    out.append((npcs, bars, tma, stores, data))
            elif ins[0] == "arrive":
                out.append((npcs, self._arrive(bars, ins[1]), tma, stores, data))
            elif ins[0] == "tma":
                d = dict(data)
                ins[2](d, "issue")
                out.append((npcs, bars, tma + ((ins[1], ins[2]),), stores, tuple(sorted(d.items()))))
            elif ins[0] == "do":
                d = dict(data)
                ins[1](d)
                out.append((npcs, bars, tma, stores, tuple(sorted(d.items()))))
            elif ins[0] == "store":
                w, buf = ins[1], ins[2]
                n, fl = stores[w]
                ns = stores[:w] + ((n + 1, fl + ((n, buf),)),) + stores[w + 1:]
                out.append((npcs, bars, tma, ns, data))
            elif ins[0] == "check_buf":
                w, b = ins[1], ins[2]
                assert all(g[1] != b for g in stores[w][1]), f"warpgroup {w} rewrites staging buffer {b} while a TMA store reads it"
                out.append((npcs, bars, tma, stores, data))
            elif ins[0] == "wait_read":
                w, n = ins[1], ins[2]
                if all(g[0] >= stores[w][0] - n for g in stores[w][1]):      # all but the n most recent bulk groups have read smem
                    out.append((npcs, bars, tma, stores, data))
        for k, (b, fn) in enumerate(tma):                                     # any in-flight TMA load lands
            d = dict(data)
            fn(d, "land")
            out.append((pcs, self._arrive(bars, b), tma[:k] + tma[k + 1:], stores, tuple(sorted(d.items()))))
        for w in range(2):                                                    # any in-flight bulk group finishes reading
            n, fl = stores[w]
            for k in range(len(fl)):
                ns = stores[:w] + ((n, fl[:k] + fl[k + 1:]),) + stores[w + 1:]
                out.append((pcs, bars, tma, ns, data))
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
                assert not stuck and not st[2] and not any(f for _, f in st[3]), f"deadlock: {stuck}"
            for t in nxt:
                if t not in seen:
                    seen.add(t)
                    stack.append(t)
        return len(seen)


def named(name, fn):
    fn.__name__ = name
    return fn


def pingpong_model(units, num_k, n_stages, mutant=None):
    """`units` = the CTA's units (sequence indices 0 .. units - 1), each of `num_k` k-blocks, through a ring of `n_stages` stages."""
    data = {"issued": 0}
    for s in range(n_stages):
        data[f"st{s}"], data[f"st{s}_readers"] = None, 0
    for w in range(2):
        for b in range(NBUF):
            data[f"buf{w}_{b}"] = None

    def tma(s, i, kb):
        def fn(d, what):
            if what == "issue":
                assert d[f"st{s}_readers"] == 0, f"TMA overwrites stage {s} ({d[f'st{s}']}) while it is read, with {(i, kb)}"
                d[f"st{s}"] = None
            else:
                d[f"st{s}"] = (i, kb)
        return named(f"tma{s}_{i}_{kb}", fn)

    def read_begin(w, i, kb, s):
        def fn(d):
            assert d[f"st{s}"] == (i, kb), f"warpgroup {w} unit {i} k-block {kb} reads stage {s} holding {d[f'st{s}']}"
            d[f"st{s}_readers"] += 1
        return named(f"read{w}_{i}_{kb}", fn)

    def read_end(s):
        def fn(d):
            d[f"st{s}_readers"] -= 1
        return named(f"release{s}", fn)

    def mainloop_begin(w, i):
        def fn(d):
            assert d["issued"] == i, f"warpgroup {w} starts unit {i} while unit {d['issued']} is still issuing"
        return named(f"begin{w}_{i}", fn)

    def mainloop_end(i):
        def fn(d):
            d["issued"] = i + 1
        return named(f"end{i}", fn)

    def stage_write(w, b, q, i):
        def fn(d):
            d[f"buf{w}_{b}"] = (i, q)
        return named(f"stage{w}_{b}_{i}_{q}", fn)

    # producer: every k-block of every unit of the CTA, in sequence order
    producer = []
    pos = 0
    for i in range(units):
        for kb in range(num_k):
            s, ph = pos % n_stages, (pos // n_stages) & 1
            producer += [("wait", f"empty{s}", ph if mutant == "empty_parity" else ph ^ 1), ("tma", f"full{s}", tma(s, i, kb))]
            pos += 1
    roles = {"producer": producer}
    # consumers: warpgroup w takes units w, w + 2, ...
    for w in range(2):
        prog = []
        for i in range(w, units, 2):
            if i > 0:
                parity = ((i >> 1) & 1) if mutant == "turn_parity" else (((i - 1) >> 1) & 1)
                prog += [("wait", f"turn{w}", parity)]
            prog += [("do", mainloop_begin(w, i))]
            pos = (i // 2) * num_k if mutant == "first_stage" else i * num_k
            prev = None
            for kb in range(num_k):
                s, ph = pos % n_stages, (pos // n_stages) & 1
                prog += [("wait", f"full{s}", ph), ("do", read_begin(w, i, kb, s))]
                if prev is not None:                      # wgmma_wait<1>: the previous stage's wgmmas retired
                    prog += [("do", read_end(prev)), ("arrive", f"empty{prev}")]
                prev = s
                pos += 1
            prog += [("do", mainloop_end(i))]
            if mutant != "no_turn_arrive":
                prog += [("arrive", f"turn{1 - w}")]
            prog += [("do", read_end(prev)), ("arrive", f"empty{prev}")]
            for q in range(NSUB):                         # epilogue: sub-tile q through staging buffer q % 2
                b = q % NBUF
                prog += [("wait_read", w, 2 if mutant == "wait_read_2" else 1), ("check_buf", w, b), ("do", stage_write(w, b, q, i)),
                         ("store", w, b)]
        prog += [("wait_read", w, 0)]
        roles[f"warpgroup{w}"] = prog
    bars = {f"full{s}": 1 for s in range(n_stages)}
    bars.update({f"empty{s}": 1 for s in range(n_stages)})
    bars.update({"turn0": 1, "turn1": 1})
    return Model(roles, bars, data)


@pytest.mark.parametrize("units,num_k,n_stages", [(1, 1, 2), (1, 3, 2), (2, 1, 2), (2, 2, 3), (3, 1, 2), (3, 2, 2), (4, 1, 3), (4, 2, 3),
                                                  (5, 1, 2)])
def test_pingpong_protocol(units, num_k, n_stages):
    assert pingpong_model(units, num_k, n_stages).explore() > units * num_k


@pytest.mark.parametrize("mutant", ["no_turn_arrive", "first_stage", "turn_parity", "empty_parity", "wait_read_2"])
def test_checker_catches_mutant(mutant):
    caught = False
    for units, num_k, n_stages in [(3, 1, 2), (3, 2, 3), (4, 1, 2)]:
        try:
            pingpong_model(units, num_k, n_stages, mutant=mutant).explore()
        except AssertionError:
            caught = True
            break
    assert caught, mutant
