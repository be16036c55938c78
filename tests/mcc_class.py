"""A numpy restatement of GLCM phase A's MCC classification, vectorised over many 3x3x3 windows.

Per (window, angle slot) the level graph has the levels at the ends of the angle's valid pairs (both ends non-zero) as
nodes and one edge per distinct unordered level pair.  Union-find over the graph's bipartite double cover (node
(level, parity); an edge {a, b} joins (a, 0) with (b, 1) and (a, 1) with (b, 0)) answers both questions at once: the
graph is connected when every level's (level, 0) lies in the set of (l0, 0) or of (l0, 1), and a connected graph is
bipartite when those two sets differ.  Classes (glcm_fast_angle): EMPTY (no valid pair: not counted), ONE (one level:
MCC 0), SPLIT (several components: 1), BIPARTITE (connected, 2-colourable: 1), TASK (an eigen-solve)."""
import numpy as np

from helpers import slot_angles

EMPTY, ONE, SPLIT, BIPARTITE, TASK = range(5)
NP = [18] * 3 + [12] * 6 + [8] * 4          # pairs per slot: axes, face diagonals, body diagonals


def slot_pairs(slot):
    """window positions (p, p + angle) of a slot, in the kernel's pair order"""
    a = slot_angles()[slot]
    return np.array([(i * 9 + j * 3 + k, (i + a[0]) * 9 + (j + a[1]) * 3 + k + a[2]) for i in range(3) for j in range(3)
                     for k in range(3) if 0 <= i + a[0] < 3 and 0 <= j + a[1] < 3 and 0 <= k + a[2] < 3]).T


def _find(par, rows, x):
    while True:
        p = par[rows, x]
        if np.array_equal(p, x):
            return x
        x = p


def classify(windows, slot):
    """windows: (V, 27) levels (0 = outside the ROI or the volume).  Returns per window the class, the node count nlev,
    the valid pair count n and the number of distinct level pairs (graph edges, self-loops included)."""
    W = np.asarray(windows, np.int64)
    V = W.shape[0]
    pa, pb = slot_pairs(slot)
    a, b = W[:, pa], W[:, pb]
    valid = (a > 0) & (b > 0)
    n = valid.sum(1)
    L = int(W.max()) + 1
    rows = np.arange(V)
    par = np.tile(np.arange(2 * L), (V, 1))
    for t in range(pa.size):
        v = valid[:, t]
        for x, y in ((a[:, t], b[:, t] + L), (a[:, t] + L, b[:, t])):
            rx, ry = _find(par, rows, x), _find(par, rows, y)
            lo, hi = np.minimum(rx, ry), np.maximum(rx, ry)
            par[rows[v], hi[v]] = lo[v]
    ends = np.concatenate([np.where(valid, a, 0), np.where(valid, b, 0)], 1)
    present = np.zeros((V, L), bool)
    present[np.repeat(rows, ends.shape[1]), ends.ravel()] = True
    present[:, 0] = False
    nlev = present.sum(1)
    l0 = np.argmax(present, 1)                   # the lowest level of the graph
    r0, r1 = _find(par, rows, l0), _find(par, rows, l0 + L)
    conn = np.ones(V, bool)
    for lev in range(1, L):
        r = _find(par, rows, np.full(V, lev))
        conn &= ~present[:, lev] | (r == r0) | (r == r1)
    codes = np.where(valid, np.minimum(a, b) * 65536 + np.maximum(a, b), -1)
    s = np.sort(codes, 1)
    edges = ((np.diff(s, axis=1) != 0) & (s[:, 1:] >= 0)).sum(1) + (s[:, 0] >= 0)
    cls = np.full(V, TASK)
    cls[conn & (r0 != r1)] = BIPARTITE
    cls[~conn] = SPLIT
    cls[nlev == 1] = ONE
    cls[n == 0] = EMPTY
    return cls, nlev, n, edges


def windows_of(lev, centres):
    """(V, 27) windows of the given centres (an (V, 3) array of z, y, x) of a level volume, 0 beyond its faces"""
    pad = np.pad(np.asarray(lev, np.int64), 1)
    z, y, x = np.asarray(centres).T
    return np.stack([pad[z + dz, y + dy, x + dx] for dz in range(3) for dy in range(3) for dx in range(3)], 1)
