"""Seeded random query trees holding ConstantScoreQuery and MinScoreQuery nodes. TEST INFRASTRUCTURE ONLY.

query_gen.Generator's space, leaves, boosts and limits (depth 4, 8 nested nodes, 32 clauses, 8 term slots), with the two
wrappers added at every depth, under every occur, inside dismaxes, nested in each other and at the root. A wrapper holds
a leaf or a nested node. A MinScoreQuery's threshold comes from threshold(inner, rng), which the caller draws from the
exact scores of the docs the inner query matches, so docs on the equality boundary are exercised."""
import numpy as np

import query_gen as qg
from nrtsearch_b200.search import BooleanQuery, BoostQuery, ConstantScoreQuery, DisjunctionMaxQuery, MinScoreQuery


class ScoreNodeGenerator(qg.Generator):
    def __init__(self, space: qg.Space, seed: int, threshold):
        super().__init__(space, seed)
        self.threshold = threshold

    def node(self, depth: int, bud, used: list, dismax: bool):
        n = int(self.rng.integers(1, 6))
        children = []
        for _ in range(n):
            if bud.clauses >= qg.MAX_CLAUSES:
                break
            r = self.rng.random()
            room = depth < qg.MAX_DEPTH and bud.nodes < qg.MAX_NODES
            if room and r < 0.25 and bud.clauses + 2 <= qg.MAX_CLAUSES:
                bud.nodes += 1
                bud.clauses += 1
                sub = self.boosted(self.wrapper(depth + 1, bud, used))
            elif room and r < 0.45:
                bud.nodes += 1
                bud.clauses += 1
                sub = self.boosted(self.node(depth + 1, bud, used, self.rng.random() < 0.35))
            else:
                sub = self.leaf(bud, used, True)
            children.append(sub)
        if dismax:
            return DisjunctionMaxQuery(children, qg.TIES[self.rng.integers(len(qg.TIES))])
        return self._bool(children)

    def wrapper(self, depth: int, bud, used: list):
        """a wrapper node at `depth` (the caller has counted the node and its clause in the parent; there is room for
        the wrapper's own clause)"""
        r = self.rng.random()
        if depth < qg.MAX_DEPTH and bud.nodes < qg.MAX_NODES and r < 0.5:
            bud.nodes += 1
            bud.clauses += 1
            if r < 0.15 and bud.clauses < qg.MAX_CLAUSES:
                inner = self.wrapper(depth + 1, bud, used)
            else:
                inner = self.node(depth + 1, bud, used, self.rng.random() < 0.35)
            inner = self.boosted(inner)
        else:
            inner = self.leaf(bud, used, True)
        if self.rng.random() < 0.5:
            return ConstantScoreQuery(inner)
        return MinScoreQuery(inner, self.threshold(inner, self.rng))

    def tree_query(self):
        if self.rng.random() < 0.15:   # a wrapper at the root
            bud = qg._Budget()
            bud.nodes, bud.clauses = 1, 1
            return self.boosted(self.wrapper(2, bud, []), root=True)
        return super().tree_query()

    def query(self):
        return self.tree_query()


def wrappers(q) -> list:
    """the ConstantScoreQuery / MinScoreQuery objects of q, outermost first"""
    out = []
    while isinstance(q, BoostQuery):
        q = q.query
    if isinstance(q, (ConstantScoreQuery, MinScoreQuery)):
        out.append(q)
        out += wrappers(q.filter if isinstance(q, ConstantScoreQuery) else q.query)
    elif isinstance(q, BooleanQuery):
        for c in q.clauses:
            out += wrappers(c.query)
    elif isinstance(q, DisjunctionMaxQuery):
        for d in q.disjuncts:
            out += wrappers(d)
    return out


def threshold_from(ref):
    """threshold(inner, rng) over an object-level reference ref (score_nodes_reference.ScoreNodeReference): mostly the exact score of a live doc the inner query
    matches, or its next float up; sometimes NaN, 0 (compiled as the inner query) or a fixed value"""
    def draw(inner, rng):
        p, s = ref.eval(inner)
        m = s[p & ref.live]
        r = rng.random()
        if r < 0.06:
            return float("nan")
        if r < 0.12:
            return 0.0
        if len(m) == 0 or r < 0.22:
            return float((1e-3, 0.7, 2.5, 1e30)[rng.integers(4)])
        v = np.float32(m[rng.integers(len(m))])
        if r < 0.32:
            v = np.nextafter(v, np.float32(np.inf))
        return float(v)
    return draw
