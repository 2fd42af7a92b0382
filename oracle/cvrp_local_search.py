"""TEST INFRASTRUCTURE ONLY -- NumPy float32 restatement of the CVRP local search of ``co_cvrp_local_search``
(include/corollout.h states the search).  ``swapstar`` has the signature of the reference's
``rl4co/envs/routing/cvrp/local_search.py:swapstar``, so it can stand in for the HGS call there:

  demands  [N+1] float32, the depot's 0 in front (customers already divided by the capacity)
  matrix   [N+1, N+1] float32, used as given
  positions  ignored (the matrix carries the distances)
  routes   list of [0, c..., 0] arrays, one per slot
  count    most moves to apply

It returns one ``[0, c..., 0]`` array per slot, in slot order (``[0, 0]`` for a slot a move emptied).

Every arithmetic operation is one float32 NumPy operation in the order the header parenthesises, so its result is the
round-to-nearest value the kernel's ``__fadd_rn`` / ``__fsub_rn`` produce.  A sweep scores all candidates at once as
[M, M] arrays over the ids 1..M (customers 1..N, then the start depot N+1+r of slot r) and takes the first minimum in
(kind, u, v) order.
"""

from __future__ import annotations

import numpy as np

RELOCATE, SWAP, TWO_OPT, TWO_OPT_STAR = 0, 1, 2, 3


def _state(slots, dem, N):
    """pred / succ / route / position per id (customers, start depots N+1+r, end depots 2N+1+r), prefix loads and
    route loads, the loads as float32 left-to-right sums in route order."""
    E = 3 * N + 1
    pred, succ = np.zeros(E, np.int64), np.zeros(E, np.int64)
    route, pos = np.full(E, -1, np.int64), np.zeros(E, np.int64)
    pref = np.zeros(E, np.float32)
    load = np.zeros(len(slots), np.float32)
    for r, cust in enumerate(slots):
        chain = [N + 1 + r, *cust, 2 * N + 1 + r]
        acc = np.float32(0)
        for k, x in enumerate(chain):
            route[x], pos[x] = r, k
            if k > 0:
                pred[x] = chain[k - 1]
            if k + 1 < len(chain):
                succ[x] = chain[k + 1]
            if 0 < k < len(chain) - 1:
                acc = np.float32(acc + dem[x])
                pref[x] = acc
        load[r] = acc
    return pred, succ, route, pos, pref, load


def best_move(slots, dem, d, capacity=1.0):
    """(delta, kind, u, v) of the smallest admissible key of one sweep, or None when it is not below -1e-6."""
    N = d.shape[0] - 1
    R = len(slots)
    M = N + R
    lim = np.float32(np.float32(capacity) + np.float32(1e-5))
    pred, succ, route, pos, pref, load = _state(slots, dem, N)
    node = np.arange(3 * N + 1)
    node[node > N] = 0  # a depot id reads row / column 0
    ids = np.arange(1, M + 1)
    u, v = ids[:, None], ids[None, :]
    pu, su, ru, qu = pred[u], succ[u], route[u], pos[u]
    pv, sv, rv, qv = pred[v], succ[v], route[v], pos[v]
    demn = np.concatenate([dem, np.zeros(2 * N, np.float32)])  # 0 for depot ids
    du, dv = demn[u], demn[v]
    lu, lv = load[ru], load[rv]

    def D(a, b):
        return d[node[a], node[b]]

    same = ru == rv
    inf = np.float32(np.inf)
    cand = np.full((4, M, M), inf, np.float32)

    rem = (D(pu, su) - D(pu, u)) - D(u, su)
    ins = (D(v, u) + D(u, sv)) - D(v, sv)
    ok = (u <= N) & (v != u) & (v != pu)
    ok &= np.where(same, lu <= lim, ((lu - du) <= lim) & ((lv + du) <= lim))
    cand[RELOCATE] = np.where(ok, rem + ins, inf)

    a = ((D(pu, v) + D(v, su)) - D(pu, u)) - D(u, su)
    c = ((D(pv, u) + D(u, sv)) - D(pv, v)) - D(v, sv)
    ok = (u <= N) & (v <= N) & (u < v) & (su != v) & (sv != u)
    ok &= np.where(same, lu <= lim, (((lu - du) + dv) <= lim) & (((lv - dv) + du) <= lim))
    cand[SWAP] = np.where(ok, a + c, inf)

    delta = ((D(u, v) + D(su, sv)) - D(u, su)) - D(v, sv)
    ok = (v <= N) & same & (qu < qv) & (su != v) & (lu <= lim)
    cand[TWO_OPT] = np.where(ok, delta, inf)

    delta = ((D(u, sv) + D(v, su)) - D(u, su)) - D(v, sv)
    ok = (ru < rv) & ((u <= N) | (v <= N)) & ((su <= 2 * N) | (sv <= 2 * N))
    ok &= ((pref[u] + (lv - pref[v])) <= lim) & ((pref[v] + (lu - pref[u])) <= lim)
    cand[TWO_OPT_STAR] = np.where(ok, delta, inf)

    m = cand.min()
    if not float(m) < -1e-6:
        return None
    kind, i, j = np.unravel_index(int(np.flatnonzero(cand == m)[0]), cand.shape)
    return m, int(kind), int(i) + 1, int(j) + 1


def apply_move(slots, N, kind, u, v):
    """Apply move (kind, u, v) to the customer lists of the slots, in place."""
    def where(x):  # (slot, index in its list; -1 for a start depot)
        if x > N:
            return x - N - 1, -1
        for r, cust in enumerate(slots):
            if x in cust:
                return r, cust.index(x)
        raise ValueError(x)

    ru, iu = where(u)
    rv, iv = where(v)
    if kind == RELOCATE:
        slots[ru].pop(iu)
        rv, iv = where(v)
        slots[rv].insert(iv + 1, u)
    elif kind == SWAP:
        slots[ru][iu], slots[rv][iv] = v, u
    elif kind == TWO_OPT:
        cust = slots[ru]
        cust[iu + 1:iv + 1] = cust[iu + 1:iv + 1][::-1]
    else:
        a, b = slots[ru], slots[rv]
        slots[ru], slots[rv] = a[:iu + 1] + b[iv + 1:], b[:iv + 1] + a[iu + 1:]


def search(slots, dem, d, count, capacity=1.0):
    """Run the search on customer lists (one per slot); returns (slots, moves applied)."""
    slots = [list(map(int, s)) for s in slots]
    dem = np.asarray(dem, np.float32)
    d = np.asarray(d, np.float32)
    N = d.shape[0] - 1
    it = 0
    while it < count:
        mv = best_move(slots, dem, d, capacity)
        if mv is None:
            break
        apply_move(slots, N, *mv[1:])
        it += 1
    return slots, it


def swapstar(demands, matrix, positions, routes, count=1, capacity=1.0):
    """Drop-in for the reference's swapstar (see the module docstring)."""
    del positions
    slots = [[int(x) for x in r if x != 0] for r in routes]
    slots, _ = search(slots, demands, matrix, count, capacity)
    return [np.array([0, *s, 0], dtype=np.int64) for s in slots]


def split_routes(tour):
    """Customer lists of a tour in the action format (maximal runs of non-zero ids, in order)."""
    slots, cur = [], []
    for x in list(np.asarray(tour).reshape(-1)) + [0]:
        if x != 0:
            cur.append(int(x))
        elif cur:
            slots.append(cur)
            cur = []
    return slots


def merge_routes(slots, width):
    """The kernel's output row: non-empty slots in order, one 0 between them, zero padding to `width`."""
    row = []
    for s in slots:
        if s:
            row += ([0] if row else []) + s
    return np.array(row + [0] * (width - len(row)), dtype=np.int64), len(row)
