"""Scheduling logic of the dataflow Cholesky kernel (chol_stream_kernel, csrc/chol.cuh), modelled on the CPU: the task decode
enumerates every lower-triangle tile exactly once, every dependency of a task belongs to an EARLIER task, and a grid of G
persistent CTAs that deal the tasks round-robin and work through them in ascending order always finishes (no spin-wait can
deadlock), for any number of tile rows and any grid size -- including far more tasks than CTAs, which the GPU tests only touch
at one size.
lookahead=True is the kernel's numbering: the diagonal tile (c+1, c+1) rides with the task of (c+1, c).  lookahead=False is the
numbering it is derived from, one task per tile in column-major order; the deadlock argument in chol.cuh (column-major
numbering, round-robin dealing, ascending order per CTA) is checked for both, so that it is seen not to rest on the merge."""
import pytest


def n_tasks(nbk, lookahead):                     # lookahead: chol_stream_tasks
    return nbk + (nbk - 1) * (nbk - 2) // 2 if lookahead else nbk * (nbk + 1) // 2


def decode(t, nbk, lookahead):
    """-> (i, c, merged): the tile (i, c) of task t; merged tasks also factor the diagonal tile (i, i)."""
    if not lookahead:                            # one task per tile, column-major over the lower triangle
        rem, c = t, 0
        while rem >= nbk - c:
            rem -= nbk - c; c += 1
        return c + rem, c, False
    if t == 0:                                   # chol_stream_kernel
        return 0, 0, False
    rem, cnt, c = t - 1, nbk - 1, 0
    while rem >= cnt:
        rem -= cnt; c += 1; cnt = nbk - 1 - c
    return c + 1 + rem, c, rem == 0


def producers(nbk, lookahead):
    """tile (a, b) -> task that publishes it."""
    prod = {}
    for t in range(n_tasks(nbk, lookahead)):
        i, c, merged = decode(t, nbk, lookahead)
        assert (i, c) not in prod
        prod[(i, c)] = t
        if merged:
            assert (i, i) not in prod
            prod[(i, i)] = t
    return prod


def deps(t, nbk, lookahead):
    i, c, merged = decode(t, nbk, lookahead)
    d = set()
    for k in range(c):                           # updates: L(i,k), L(c,k)
        d.add((i, k)); d.add((c, k))
    if i != c:
        d.add((c, c))                            # the solve needs the diagonal factor of its column
    return d


@pytest.mark.parametrize("lookahead", [False, True])
@pytest.mark.parametrize("nbk", [1, 2, 3, 4, 7, 19, 34, 61])
def test_every_tile_once_and_dependencies_point_backwards(nbk, lookahead):
    prod = producers(nbk, lookahead)
    assert set(prod) == {(i, c) for i in range(nbk) for c in range(i + 1)}
    for t in range(n_tasks(nbk, lookahead)):
        for tile in deps(t, nbk, lookahead):
            assert prod[tile] < t or (prod[tile] == t and tile != decode(t, nbk, lookahead)[:2]), (t, tile)


@pytest.mark.parametrize("lookahead", [False, True])
@pytest.mark.parametrize("nbk,grid", [(1, 1), (2, 1), (4, 3), (7, 1), (7, 5), (19, 172), (19, 13), (34, 296), (34, 7), (61, 148)])
def test_round_robin_persistent_grid_never_deadlocks(nbk, grid, lookahead):
    nt = n_tasks(nbk, lookahead)
    prod = producers(nbk, lookahead)
    queues = [list(range(g, nt, grid)) for g in range(min(grid, nt))]
    done = set()
    pos = [0] * len(queues)
    finished = 0
    while finished < nt:
        progressed = False
        for g, q in enumerate(queues):
            if pos[g] == len(q):
                continue
            t = q[pos[g]]
            if all(prod[tile] in done or prod[tile] == t for tile in deps(t, nbk, lookahead)):
                done.add(t); pos[g] += 1; finished += 1; progressed = True
        assert progressed, f"deadlock with {nt - finished} tasks left"
