"""The neighbour-warp protocol of the fused TV-L1 tile loop (denseflow_b200/csrc/tvl1_fused.cu, tile_iteration) with dead halo
warps, explored over every interleaving with the checker of test_sync_protocol_cpu.py.

Counted from a region edge that is halo, iteration `it` of a tile visit needs the primal step only on rows [it+1, TH-it) and
the dual step only on [it+1, TH-it-1).  A warp whose rows all lie outside skips the arithmetic: it reads and writes no row,
but keeps its waits and signals.  Here every warp holds one row of a W-row tile whose top and bottom edges are both halo."""
from collections import deque

from test_sync_protocol_cpu import explore, warp_programs


def dead_row_warp_programs(W, iters, dead_waits=True):
    """warp_programs with dead rows skipped.  A live warp checks a neighbour's row only where its own result is needed: the
    kernel computes its other rows from stale values, which feed dead rows only."""
    progs = []
    for w in range(W):
        p = []
        for it in range(iters):
            if not it + 1 <= w < W - it:
                if w > 0 and dead_waits:
                    p.append(("wait_ge", ("prog", w - 1), 2 * it))
                p.append(("write", ("prog", w), 2 * it + 1))
                if w < W - 1 and dead_waits:
                    p.append(("wait_ge", ("prog", w + 1), 2 * it + 1))
                p.append(("write", ("prog", w), 2 * it + 2))
                continue
            if w > 0:
                p.append(("wait_ge", ("prog", w - 1), 2 * it))
                p.append(("read", ("p_bot", w - 1), it))  # the primal step of this row is live: it needs p(it-1) of the row above
            p.append(("write", ("u_row0", w), it + 1))
            p.append(("write", ("prog", w), 2 * it + 1))
            if w < W - 1:
                p.append(("wait_ge", ("prog", w + 1), 2 * it + 1))
                if w < W - it - 1:
                    p.append(("read", ("u_row0", w + 1), it + 1))
            p.append(("write", ("p_bot", w), it + 1))
            p.append(("write", ("prog", w), 2 * it + 2))
        progs.append(p)
    return progs, warp_programs(W, iters)[1]


def test_dead_halo_warps_keep_every_live_cross_warp_read_ordered():
    for W, iters in ((5, 2), (6, 2), (7, 3)):
        v, dead, states = explore(*dead_row_warp_programs(W, iters))
        assert not v and dead == 0, (W, iters, v[:3])
        assert states > 100


def max_lead(progs, mem):
    """the largest prog[w] - prog[w +- 1] over every state the waits allow"""
    W = len(progs)
    locs = sorted(mem, key=repr)
    idx = {l: i for i, l in enumerate(locs)}
    pairs = [(idx[("prog", w)], idx[("prog", nb)]) for w in range(W) for nb in (w - 1, w + 1) if 0 <= nb < W]
    start = (tuple(0 for _ in progs), tuple(mem[l] for l in locs))
    seen, todo, best = {start}, deque([start]), 0
    while todo:
        pcs, m = todo.popleft()
        best = max([best] + [m[a] - m[b] for a, b in pairs])
        for t, prog in enumerate(progs):
            if pcs[t] == len(prog):
                continue
            op, loc, val = prog[pcs[t]]
            if op == "wait_ge" and m[idx[loc]] < val:
                continue
            mm = list(m)
            if op == "write":
                mm[idx[loc]] = val
            nxt = (pcs[:t] + (pcs[t] + 1,) + pcs[t + 1:], tuple(mm))
            if nxt not in seen:
                seen.add(nxt)
                todo.append(nxt)
    return best


def test_dead_warps_keep_their_waits_so_they_never_run_ahead_of_a_neighbour():
    """Without TMA no CTA-wide barrier separates two tiles, so a warp that finished its visit early would overwrite its rows of
    the next tile while its neighbours still read them.  With its waits a dead warp's counter leads a neighbour's by no more
    than in the live protocol; without them it can finish the whole visit first."""
    live = max_lead(*warp_programs(5, 3))
    assert max_lead(*dead_row_warp_programs(5, 3)) <= live
    assert max_lead(*dead_row_warp_programs(5, 3, dead_waits=False)) > live
