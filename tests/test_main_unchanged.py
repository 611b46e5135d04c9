"""The stand-ins under compat/ that let the reference's unmodified learning/main.py run on top of
superpoint_graph_b200 (compat/run_main.py) where igraph is not installed."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "compat"))


def test_compat_igraph_semantics():
    import igraph
    G = igraph.Graph(n=5, edges=[[0, 1], [1, 2], [3, 4], [4, 0], [2, 1]], directed=True,
                     edge_attrs={"f": [10, 11, 12, 13, 14]}, vertex_attrs={"v": list(range(5)), "s": [5, 50, 7, 70, 9]})
    assert G.indegree(G.vs, loops=True) == [1, 2, 1, 0, 1]
    S = G.subgraph([4, 0, 1])  # renumbered in increasing order of the old ids: 0->0, 1->1, 4->2
    assert S.vcount() == 3 and S.vs["v"] == [0, 1, 4] and S.get_edgelist() == [(0, 1), (2, 0)] and S.es["f"] == [10, 13]
    P = G.permute_vertices([2, 0, 1, 4, 3])  # vertex i becomes perm[i]
    assert P.vs["v"] == [1, 2, 0, 4, 3] and P.get_edgelist()[0] == (2, 0) and P.es["f"] == G.es["f"]
    assert sorted(G.neighborhood([3], 2)[0]) == [0, 3, 4] and G.neighborhood([3], 1)[0][0] == 3
    sub = G.es[[4, 0]]
    assert sub.get_attribute_values("f") == [14, 10] and G.vs[3]["s"] == 70
