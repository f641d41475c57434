"""The linear-sum-assignment solver as the native kernel runs it, in plain Python: scipy's rectangular_lsap.cpp
(shortest augmenting paths, Crouse 2016) restated step for step in float64, with the column selection written
as the kernel's parallel argmin rather than scipy's sequential scan.

    solve(cost) -> (row_ind, col_ind), what scipy.optimize.linear_sum_assignment(cost) returns
    solve_matching(cost) -> (col4row, row4col, steps), the kernel's outputs (-1 for unmatched) and the Dijkstra
                            steps it takes

The column picked at each step is, among the remaining columns of least shortest-path cost, the one with the
largest position in `remaining` that is unassigned if there is any, else the one with the smallest position
(the kernel minimises the key (spc, unassigned ? -it : it + 2^30)).  scipy's scan (update on spc < lowest, or on
spc == lowest for an unassigned column) selects the same column."""
import numpy as np


class Infeasible(ValueError):
    pass


def solve_matching(cost):
    cost = np.asarray(cost, np.float64)
    R, C = cost.shape
    if np.isnan(cost).any() or (cost == -np.inf).any():
        raise ValueError("matrix contains invalid numeric entries")
    tr = C < R
    a = cost.T if tr else cost
    nr, nc = a.shape
    u, v = np.zeros(nr), np.zeros(nc)
    col4row, row4col, path = -np.ones(nr, int), -np.ones(nc, int), -np.ones(nc, int)
    steps = 0
    for cur in range(nr):
        spc = np.full(nc, np.inf)
        SR, SC = np.zeros(nr, bool), np.zeros(nc, bool)
        remaining = np.arange(nc - 1, -1, -1)
        num_remaining = nc
        i, min_val, sink = cur, 0.0, -1
        while sink == -1:
            steps += 1
            SR[i] = True
            rem = remaining[:num_remaining]
            r = ((min_val + a[i, rem]) - u[i]) - v[rem]          # every entry rounded as the kernel does
            upd = r < spc[rem]
            path[rem[upd]] = i
            spc[rem[upd]] = r[upd]
            vals = spc[rem]
            lowest = vals.min()
            if lowest == np.inf:
                raise Infeasible("cost matrix is infeasible")
            tied = np.nonzero(vals == lowest)[0]                  # positions `it` of the least path cost
            free = tied[row4col[rem[tied]] == -1]
            it = free.max() if len(free) else tied.min()
            min_val = lowest
            j = remaining[it]
            if row4col[j] == -1:
                sink = j
            else:
                i = row4col[j]
            SC[j] = True
            num_remaining -= 1
            remaining[it] = remaining[num_remaining]
        u[cur] += min_val
        for r in range(nr):
            if SR[r] and r != cur:
                u[r] += min_val - spc[col4row[r]]
        for c in range(nc):
            if SC[c]:
                v[c] -= min_val - spc[c]
        j = sink
        while True:
            r = path[j]
            row4col[j] = r
            col4row[r], j = j, col4row[r]
            if r == cur:
                break
    if tr:
        return row4col, col4row, steps
    return col4row, row4col, steps


def solve(cost):
    col4row, _, _ = solve_matching(cost)
    rows = np.nonzero(col4row >= 0)[0]
    return rows, col4row[rows]
