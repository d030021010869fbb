"""Exhaustive interleaving check of the clipped round's cross-GPU protocol (csrc/rs_adam_ag.cu: round_gate_kernel, round_norm_kernel,
rs_adam_ag_kernel's end barrier), in the style of test_round_protocol_model.py.

Program of a rank, round e (one line = one atomic step; `for q` lines are separate steps per peer, in any order):
    G1q pad[q].count[me] = my count of round e             (st.relaxed.sys)
    G2q pad[q].start[me] = e                               (st.release.sys, after G1q)
    G3  wait pad[me].start[*] >= e
    N1q pad[q].part[me]  = my partial sum of squares of round e   (st.relaxed.sys)
    N2q pad[q].nflag[me] = e                                (st.release.sys, after N1q)
    N3  wait pad[me].nflag[*] >= e
    N4  read pad[me].part[*], sum in rank order            -> must be every peer's round-e partial
    E1q pad[q].end[me] = e                                 (rs_adam_ag_kernel's end barrier, after the update)
    E2  wait pad[me].end[*] >= e
and the next round starts.  Checked: no deadlock, each rank reads the round-e partial of every peer (never e-1 or e+1), no partial is
overwritten before its reader has read it, and every rank derives the same norm for every round."""
import pytest

ROUNDS = 3


def part_of(rank, e):
    return 100 * e + rank + 1          # distinct per (rank, round): a stale or early read is detectable


def initial(W):
    ranks = tuple((1, "G1", frozenset(range(W))) for _ in range(W))
    zero = tuple(0 for _ in range(W))
    pads = tuple((zero, zero, zero, zero) for _ in range(W))    # start, end, part, nflag
    read = tuple(0 for _ in range(W))                          # last round whose partials rank me has read
    norms = tuple(() for _ in range(W))
    return ranks, pads, read, norms


def successors(state, W, flag_first=False, norm_wait=True):
    ranks, pads, read, norms = state
    out = []
    peers = frozenset(range(W))
    for me, (e, pc, pend) in enumerate(ranks):
        if e > ROUNDS:
            continue

        def nxt_state(rank, new_pads=pads, new_read=read, new_norms=norms):
            r = list(ranks)
            r[me] = rank
            out.append((tuple(r), new_pads, new_read, new_norms))

        order = {"G1": "G2", "G2": "G3", "N1": "N2", "N2": "N3", "E1": "E2"}
        if pc in ("G1", "G2", "N1", "N2", "E1"):
            for q in pend:
                p = [list(map(list, x)) for x in pads]
                if pc == "G1":
                    pass                                            # the count store (checked in test_round_protocol_model.py)
                elif pc == "G2":
                    p[q][0][me] = e
                elif pc == "E1":
                    p[q][1][me] = e
                elif (pc == "N1") != flag_first:                    # the value store
                    old = pads[q][2][me]
                    assert old == 0 or read[q] >= (old - me - 1) // 100, \
                        f"rank {me} overwrites its round-{(old - me - 1) // 100} partial in rank {q}'s pad before {q} read it"
                    p[q][2][me] = part_of(me, e)
                else:                                               # the flag store
                    p[q][3][me] = e
                rest = pend - {q}
                nxt = (e, pc, rest) if rest else (e, order[pc], peers if order[pc] in ("G2", "N2") else frozenset())
                nxt_state(nxt, new_pads=tuple(tuple(map(tuple, x)) for x in p))
        elif pc == "G3":
            if all(v >= e for v in pads[me][0]):
                nxt_state((e, "N1", peers))
        elif pc == "N3":
            if not norm_wait or all(v >= e for v in pads[me][3]):
                nxt_state((e, "N4", frozenset()))
        elif pc == "N4":
            got = pads[me][2]
            assert all(got[q] == part_of(q, e) for q in range(W)), f"rank {me} round {e} read partials {got}"
            rd = list(read)
            rd[me] = e
            nm = list(norms)
            nm[me] = norms[me] + (sum(got[q] for q in range(W)),)  # rank order
            nxt_state((e, "E1", peers), new_read=tuple(rd), new_norms=tuple(nm))
        elif pc == "E2":
            if all(v >= e for v in pads[me][1]):
                nxt_state((e + 1, "G1", peers))
    return out


def explore(W, **kw):
    start = initial(W)
    seen, stack, finals = {start}, [start], 0
    while stack:
        s = stack.pop()
        nxt = successors(s, W, **kw)
        if not nxt:
            assert all(e > ROUNDS for e, _, _ in s[0]), f"deadlock: {s[0]}"
            assert len(set(s[3])) == 1 and len(s[3][0]) == ROUNDS, f"ranks derived different norms: {s[3]}"
            finals += 1
        for t in nxt:
            if t not in seen:
                seen.add(t)
                stack.append(t)
    return len(seen), finals


@pytest.mark.parametrize("W,rounds", [(2, 4), (3, 2)])
def test_norm_exchange_is_safe_and_live_under_every_interleaving(W, rounds):
    global ROUNDS
    old, ROUNDS = ROUNDS, rounds
    try:
        states, finals = explore(W)
    finally:
        ROUNDS = old
    assert finals >= 1
    assert states > (500 if W == 2 else 5000)            # the exploration really branched


@pytest.mark.parametrize("broken", [dict(flag_first=True), dict(norm_wait=False)])
def test_the_checker_catches_a_broken_norm_exchange(broken):
    """The flag published before the value, or no wait for the peers' flags: some interleaving reads a stale partial."""
    with pytest.raises(AssertionError):
        explore(2, **broken)
