# -*- coding: utf-8 -*-
"""A model of the row draws of the reference's ACA (hodlr.h:178-183), written from the published algorithms and not
from the device code: the mt19937 words of a 32-bit seed, libstdc++ >= 11's ``uniform_int_distribution<int>(0, s - 1)``
on a 32-bit engine (Lemire's multiply-shift, rejecting while ``low < (2^32 - s) % s``) and the swap-pop of the row index
list.  ``tests/test_aca_draw_model.py`` pins it against the real libstdc++ through the oracle.

On top of the draws, ``predict_node`` gives everything ``low_rank_approx`` (hodlr.h:136-221) decides for a block that is
a partial permutation pattern: at most one non-zero per row and per column (``tests/test_gpu_hodlr_draws.py`` builds
such blocks).  There a candidate row is usable iff its one entry is >= 1e-14 in magnitude, the factors already found
never change another row's residual, and the cross terms of the stopping rule (hodlr.h:206-213) are exactly 0.
"""

import numpy as np

GOLDEN = 0x9E3779B9
MASK32 = 0xFFFFFFFF


def mt19937_words(seed, n):
    """The first n tempered 32-bit outputs of mt19937 seeded with init_genrand(seed), as std::mt19937::seed does.
    numpy's legacy RandomState seeds the same way, and a draw over the full 32-bit range returns the raw words."""
    rs = np.random.RandomState(int(seed) & MASK32)
    return rs.randint(0, 2 ** 32, size=int(n), dtype=np.uint64).astype(np.uint32) if n else np.zeros(0, np.uint32)


def node_seed(seed, pre_id):
    """Seed of the private stream of the node with pre-order index pre_id (per-node RNG mode)."""
    return (int(seed) + GOLDEN * int(pre_id)) & MASK32


def uniform_draws(words, sizes):
    """uniform_int_distribution<int>(0, sizes[c] - 1) for c = 0, 1, ... on the stream `words`.
    Returns (k, cum, rejected): the draws, the words consumed up to and including draw c, and one entry per rejected
    word holding the index of the draw that rejected it."""
    sizes = np.asarray(sizes, dtype=np.uint64)
    n = len(sizes)
    k = np.zeros(n, dtype=np.int64)
    cum = np.zeros(n, dtype=np.int64)
    rejected = []
    thr = (np.uint64(2 ** 32) - sizes) % sizes
    c, pos = 0, 0
    while c < n:
        m = n - c
        prod = words[pos:pos + m].astype(np.uint64) * sizes[c:]
        rej = (prod & np.uint64(MASK32)) < thr[c:]
        j = int(np.argmax(rej)) if rej.any() else m
        k[c:c + j] = (prod[:j] >> np.uint64(32)).astype(np.int64)
        cum[c:c + j] = pos + 1 + np.arange(j)
        c += j
        pos += j
        if c < n:  # draw c rejects its first word: one word at a time until one is accepted
            s, t = int(sizes[c]), int(thr[c])
            while True:
                p = int(words[pos]) * s
                pos += 1
                if (p & MASK32) >= t:
                    break
                rejected.append(c)
            k[c], cum[c] = p >> 32, pos
            c += 1
    return k, cum, rejected


def words_needed(n_rows):
    """Enough words for every draw of a node of n_rows rows, rejections included (64 spare: a node expects
    n_rows^2 / 2^33 of them)."""
    return int(n_rows) + 64


class Draws(object):
    """All n_rows draws of one node from the stream `words` (which starts at the node's first word): `rows[c]` is the
    row visited by draw c, `cum[c]` the words consumed up to and including it, `rejected` the draws that rejected a
    word (repeated when a draw rejects twice)."""

    def __init__(self, words, n_rows, order=True):
        self.n_rows = int(n_rows)
        sizes = np.arange(n_rows, 0, -1)
        self.k, self.cum, self.rejected = uniform_draws(words, sizes)
        self.rows = None
        if order:
            index = list(range(n_rows))
            rows = np.zeros(n_rows, dtype=np.int64)
            for c, kc in enumerate(self.k.tolist()):  # hodlr.h:179-183
                rows[c] = index[kc]
                index[kc] = index[-1]
                index.pop()
            self.rows = rows

    def rejections_up_to(self, c):
        return sum(1 for r in self.rejected if r <= c)


def tree(n, min_size):
    """The nodes of the HODLR tree in pre-order (hodlr.h:29-66): dicts with start, size, half, is_leaf."""
    out = []

    def build(start, size):
        half = size // 2
        nd = dict(start=start, size=size, half=half, is_leaf=not half >= min_size)
        out.append(nd)
        if not nd["is_leaf"]:
            build(start, half)
            build(start + half, size - half)
    build(0, n)
    return out


def predict_node(draws, n_rows, n_cols, special, tol):
    """The outcome of low_rank_approx on a partial-permutation block.  `special`: block row -> (block column, value).
    Returns dict(rank, rows, cols, rng_draws, dense_fallback); rng_draws counts mt19937 words."""
    max_rank = min(n_rows, n_cols)
    rows, cols = [], []
    norm = 0.0
    for c, row in enumerate(draws.rows.tolist()):
        if row not in special:
            continue
        col, a = special[row]
        if abs(a) < 1e-14:
            continue  # hodlr.h:191
        rows.append(row)
        cols.append(col)
        if len(rows) >= max_rank:
            return dict(rank=len(rows), rows=rows, cols=cols, rng_draws=int(draws.cum[c]), dense_fallback=0)
        rowcol = (a * a) * 1.0  # |u|^2 |v|^2: u is the column (one entry a), v the row over its pivot (one entry 1)
        if rowcol < tol * tol * norm:
            return dict(rank=len(rows), rows=rows, cols=cols, rng_draws=int(draws.cum[c]), dense_fallback=0)
        norm += rowcol
    return dict(rank=len(rows), rows=rows, cols=cols, rng_draws=int(draws.cum[-1]), dense_fallback=1)


def predict_tree(n, min_size, seed, specials, tol, chained=False, order_all=False):
    """predict_node for every internal node.  `specials`: pre-order index -> {block row: (block column, value)}.
    chained = False: every node draws from its own stream, node_seed(seed, pre_id); True: one stream seeded with `seed`
    runs through the internal nodes in pre-order, each starting where the previous one stopped."""
    nodes = tree(n, min_size)
    out = {}
    stream = mt19937_words(seed, sum(words_needed(nd["size"] - nd["half"]) for nd in nodes if not nd["is_leaf"])) \
        if chained else None
    offset = 0
    for i, nd in enumerate(nodes):
        if nd["is_leaf"]:
            continue
        n_rows, n_cols = nd["size"] - nd["half"], nd["half"]
        w = stream[offset:] if chained else mt19937_words(node_seed(seed, i), words_needed(n_rows))
        sp = specials.get(i, {})
        d = Draws(w, n_rows, order=bool(sp) or order_all)
        if sp:
            out[i] = predict_node(d, n_rows, n_cols, sp, tol)
        else:  # every row is rejected
            out[i] = dict(rank=0, rows=[], cols=[], rng_draws=int(d.cum[-1]), dense_fallback=1)
        out[i]["draws"] = d
        offset += out[i]["rng_draws"]
    return nodes, out


# ---- problems whose ACA outcome is a pure function of the draw order -------------------------------------------------
SPACING = 64.0       # base points, in length scales of ExpSquaredKernel(1.0): exp(-0.5 * 47^2) underflows to exactly 0
NORMAL = (0.5, 0.6, 0.7, 0.8)
TERMINATOR = 1e-12   # accepted (>= 1e-14); a^2 < tol^2 * norm then stops the node at this draw
SUB_THRESHOLD = 5e-15   # rejected by the 1e-14 test ...
AT_THRESHOLD = 2e-14    # ... and accepted, a factor of 2 on either side


class Schedule(object):
    """The device's batch schedule, used ONLY to decide where to put special rows (never in an assertion): B starts at 4,
    grows 8-fold up to bmax after a fully rejected batch, becomes 1 after an accept at position 0 and min(B, 2 (p + 1))
    after one at position p; a batch is cut to the rows left, and before a last draw that rejects a word."""

    def __init__(self, n_rows, rejected=()):
        self.n_rows, self.rejected = n_rows, set(rejected)
        self.bmax = min(8192, n_rows)
        self.first, self.B = 0, 4

    def size(self):
        b = min(self.B, self.bmax, self.n_rows - self.first)
        if b > 1 and self.first + b - 1 in self.rejected:
            b -= 1
        return b

    def reject(self):
        self.first += self.size()
        self.B = min(8 * self.B, 8192)

    def reject_until(self, draw=None, size=None):
        """Reject whole batches until the pending one contains `draw` / holds `size` candidates."""
        while (draw is not None and self.first + self.size() <= draw) or (size is not None and self.size() != size):
            assert self.first < self.n_rows
            self.reject()
        return self

    def accept(self, p):
        """Accept position p of the pending batch; returns the draw index."""
        assert 0 <= p < self.size()
        draw = self.first + p
        self.B = 1 if p == 0 else max(1, min(self.B, 2 * (p + 1)))
        self.first = draw + 1
        return draw

    def accept_draw(self, draw):
        self.reject_until(draw=draw)
        return self.accept(draw - self.first)


class Problem(object):
    """ExpSquaredKernel(1.0) on points SPACING apart, so that every off-diagonal kernel value is exactly 0, plus disjoint
    special pairs (i, j): x_j is moved to x_i + delta with k(x_i, x_j) = a.  `place(node, draw, a)` makes the row that
    draw number `draw` of `node` visits special."""

    def __init__(self, n, min_size, seed, tol=1e-10, chained=False, ndim=1):
        self.n, self.min_size, self.seed, self.tol, self.chained, self.ndim = n, min_size, seed, tol, chained, ndim
        self.nodes = tree(n, min_size)
        self.coord = SPACING * np.arange(n, dtype=np.float64)
        self.partner = -np.ones(n, dtype=np.int64)
        self.pairs = {}      # node -> list of (block row, block column, requested a)
        self.values = None

    def draws(self, node):
        """The node's draws.  Chained streams: depends on what every earlier node consumed, so place in pre-order."""
        nd = self.nodes[node]
        assert not nd["is_leaf"]
        if self.chained:
            return predict_tree(self.n, self.min_size, self.seed, self.specials(), self.tol, True, order_all=True)[1][node]["draws"]
        return Draws(mt19937_words(node_seed(self.seed, node), words_needed(nd["size"] - nd["half"])), nd["size"] - nd["half"])

    def place(self, node, draw, a, draws=None):
        nd = self.nodes[node]
        row = int((draws or self.draws(node)).rows[draw])
        gi = nd["start"] + nd["half"] + row
        assert self.partner[gi] < 0, "row already special"
        free = np.flatnonzero(self.partner[nd["start"]:nd["start"] + nd["half"]] < 0)
        col = int(free[(7919 * (draw + 1)) % len(free)])
        gj = nd["start"] + col
        self.partner[gi], self.partner[gj] = gj, gi
        self.coord[gj] = self.coord[gi] + np.sqrt(-2.0 * np.log(a))
        self.pairs.setdefault(node, []).append((row, col, a))
        self.values = None
        return row

    @property
    def x(self):
        if self.ndim == 1:
            return self.coord[:, None].copy()
        return np.stack([self.coord] + [np.zeros(self.n)] * (self.ndim - 1), axis=1)

    def kernel(self):
        from george_b200 import kernels
        return kernels.ExpSquaredKernel(1.0, ndim=self.ndim)

    def specials(self):
        """node -> {row: (col, value)} with the values the oracle's kernel gives at the moved points."""
        if self.values is None:
            import oracle
            from george_b200._spec import flatten
            spec, x = flatten(self.kernel()), self.x
            self.values = {}
            for node, lst in self.pairs.items():
                nd = self.nodes[node]
                gi = np.array([nd["start"] + nd["half"] + r for r, _, _ in lst])
                gj = np.array([nd["start"] + c for _, c, _ in lst])
                v = oracle.value_diagonal(spec, x[gi], x[gj])
                assert np.allclose(v, [a for _, _, a in lst], rtol=1e-6)
                self.values[node] = dict((r, (c, float(val))) for (r, c, _), val in zip(lst, v))
            # off the pattern the kernel is exactly 0: neighbours in coordinate order that are not partners
            order = np.argsort(self.coord)
            lo, hi = order[:-1], order[1:]
            off = self.partner[lo] != hi
            assert np.all(np.diff(self.coord[order])[off] > 40.0)
            near = np.argsort(np.diff(self.coord[order])[off])[:64]
            assert np.all(oracle.value_diagonal(spec, x[lo[off][near]], x[hi[off][near]]) == 0.0)
        return self.values

    def predict(self):
        return predict_tree(self.n, self.min_size, self.seed, self.specials(), self.tol, self.chained)[1]

    def kept_pairs(self, pred, exhaust):
        """(i, j, a) of the pairs K_h keeps: those whose row became a pivot, and with exhaust = "dense" every pair of a
        node that ran out of rows (it stores its block densely)."""
        out = []
        for node, sp in self.specials().items():
            nd, p = self.nodes[node], pred[node]
            for row, (col, a) in sp.items():
                if row in p["rows"] or (exhaust == "dense" and p["dense_fallback"]):
                    out.append((nd["start"] + nd["half"] + row, nd["start"] + col, a))
        return out


class BlockReference(object):
    """K_h = d I + the kept pairs: 1 x 1 and 2 x 2 blocks after a symmetric permutation; longdouble."""

    def __init__(self, n, d, kept):
        LD = np.longdouble
        self.n = n
        self.d = LD(d)
        self.p = np.arange(n)
        self.a = np.zeros(n, dtype=LD)
        for i, j, a in kept:
            self.p[i], self.p[j] = j, i
            self.a[i] = self.a[j] = LD(a)
        self.det = self.d * self.d - self.a * self.a   # of the 2 x 2 block (d^2 for an unpaired point)
        paired = self.p != np.arange(n)
        self.logdet = float(np.sum(np.log(self.det[paired])) / 2 + np.sum(~paired) * np.log(self.d))
        self.cond = float(np.max((self.d + np.abs(self.a)) / (self.d - np.abs(self.a))))

    def solve(self, B):
        B = np.asarray(B, dtype=np.longdouble)
        a, det = (self.a, self.det) if B.ndim == 1 else (self.a[:, None], self.det[:, None])
        return (self.d * B - a * B[self.p]) / det
