"""The tile hand-over of the fused TV-L1 tile loop (denseflow_b200/csrc/tvl1_fused.cu, process_tile), explored over every
interleaving with the checker of test_sync_protocol_cpu.py.

No CTA-wide barrier separates two tiles of a chunk: each warp loads its own rows of the next tile as soon as it is done with
the current one, and signals `base` of the new tile.  A warp's constant rows are read by its own threads only, so they are
not modelled.  What crosses warps:
* row 0 of a warp's u: written by the warp (load, every primal step), read by the warp above in its last dual row;
* p_bot of a warp: written by the warp (load, every last dual row), read by the warp below in its first primal row.
The load of the next tile waits for the warp above to have finished its last dual step of the current tile.

The model has W warps of R rows each (tile height W * R) and the kernel's dead-warp rule: counted from a region edge that is
halo, iteration `it` needs the primal step on rows [it+1, TH-it) and the dual step on [it+1, TH-it-1); a warp whose rows all
lie outside the primal range skips the iteration but keeps its waits and signals.  A read states the version it needs only
where the row it feeds is live (stale values feed dead rows only).  Versions: tile n, after i primal (u) / dual (p) steps of
the visit = n * (kk + 1) + i."""
from test_sync_protocol_cpu import explore


def handover_programs(W, R, kk, tiles, handover_wait=True):
    """tiles: [(halo_top, halo_bot)] of the CTA's consecutive tiles in one chunk (0: that region edge is the image border)."""
    TH = W * R

    def ver(n, i):
        return n * (kk + 1) + i

    progs = []
    for w in range(W):
        p = []
        r0, r1 = R * w, R * w + R - 1  # this warp's first and last row
        for n, (top, bot) in enumerate(tiles):
            base = 1 + n * (2 * kk + 2)  # tile_base: starts at 1 (counters at 0), + 2 kk + 2 per tile
            # -------- load: this warp's rows of tile n
            if w > 0 and handover_wait:
                p.append(("wait_ge", ("prog", w - 1), base - 2))  # the warp above is done with this warp's row 0
            p.append(("write", ("u_row0", w), ver(n, 0)))
            p.append(("write", ("p_bot", w), ver(n, 0)))
            p.append(("write", ("prog", w), base))
            # -------- kk iterations
            for it in range(kk):
                plo, phi = top * (it + 1), TH - bot * it          # rows with a live primal step
                dlo, dhi = top * (it + 1), TH - bot * it - 1      # rows with a live dual step
                if r1 < plo or r0 >= phi:  # dead warp: waits and signals only
                    if w > 0:
                        p.append(("wait_ge", ("prog", w - 1), base + 2 * it))
                    p.append(("write", ("prog", w), base + 2 * it + 1))
                    if w < W - 1:
                        p.append(("wait_ge", ("prog", w + 1), base + 2 * it + 1))
                    p.append(("write", ("prog", w), base + 2 * it + 2))
                    continue
                if w > 0:
                    p.append(("wait_ge", ("prog", w - 1), base + 2 * it))  # D3 of the previous iteration of the warp above
                    if plo <= r0 < phi:
                        p.append(("read", ("p_bot", w - 1), ver(n, it)))
                p.append(("write", ("u_row0", w), ver(n, it + 1)))  # P0
                p.append(("write", ("prog", w), base + 2 * it + 1))
                if w < W - 1:
                    p.append(("wait_ge", ("prog", w + 1), base + 2 * it + 1))  # P0 of the warp below
                    if dlo <= r1 < dhi:
                        p.append(("read", ("u_row0", w + 1), ver(n, it + 1)))  # D3 needs the new u of the row below
                p.append(("write", ("p_bot", w), ver(n, it + 1)))  # D3
                p.append(("write", ("prog", w), base + 2 * it + 2))
            # -------- write-back: this warp's own rows only
        progs.append(p)
    mem = {}
    for w in range(W):
        mem[("prog", w)] = 0
        mem[("u_row0", w)] = -1  # nothing loaded yet
        mem[("p_bot", w)] = -1
    return progs, mem


TOP, MID, BOT, ALL = (0, 1), (1, 1), (1, 0), (0, 0)  # (halo_top, halo_bot) of the tile's region


def dead_warps(W, R, kk, top, bot):
    """(warp, iteration) pairs the kernel skips in one visit"""
    TH = W * R
    return {(w, it) for w in range(W) for it in range(kk) if R * w + R - 1 < top * (it + 1) or R * w >= TH - bot * it}


# (W, R, kk, tiles): tile height W * R > 2 kk, as in the kernel (64 rows, kk <= 8); dead warps at both edges
CASES = [
    (3, 1, 1, [TOP, MID, BOT]),
    (4, 1, 1, [MID, MID, MID]),
    (3, 3, 4, [MID, MID]),
    (3, 3, 4, [TOP, BOT]),
    (3, 3, 4, [MID, MID, BOT]),
    (3, 6, 8, [TOP, MID, BOT]),
    (3, 6, 8, [MID, MID]),
    (3, 6, 8, [BOT, TOP]),
    (3, 6, 8, [ALL, MID]),
]


def test_cases_have_dead_warps_at_both_edges():
    for W, R, kk, tiles in CASES:
        if kk == 1:
            continue  # the kernel has no dead warp in a one-iteration visit (4 rows per warp)
        d = dead_warps(W, R, kk, 1, 1)
        assert any(w == 0 for w, _ in d) and any(w == W - 1 for w, _ in d), (W, R, kk)


def test_tile_handover_orders_every_cross_warp_read():
    """No warp overwrites u row 0 or p_bot of tile n while a neighbour can still read it, and no warp reads a neighbour's
    rows of tile n + 1 before that neighbour has loaded them."""
    for W, R, kk, tiles in CASES:
        v, dead, states = explore(*handover_programs(W, R, kk, tiles))
        assert not v and dead == 0, (W, R, kk, tiles, v[:3])
        assert states > 100


def test_handover_without_the_wait_for_the_warp_above_overwrites_a_row_it_still_reads():
    for W, R, kk, tiles in ((3, 1, 1, [MID, MID]), (3, 3, 4, [MID, BOT, MID]), (3, 6, 8, [BOT, MID])):
        v, _, _ = explore(*handover_programs(W, R, kk, tiles, handover_wait=False))
        assert v, (W, R, kk, tiles)
        assert all(loc[0] == "u_row0" for _, _, loc, _, _ in v)
