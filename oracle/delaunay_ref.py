"""Exact 3D Delaunay triangulation of float32 clouds: the oracle of superpoint_graph_b200/spg_delaunay.py.

Two parts, both in exact arithmetic on the float32 coordinates (Python integers after scaling by 2^149):

- `certificate(xyz, simplices)` checks a triangulation without recomputing it.  Every tetrahedron has exact
  positive orientation; every interior face is shared by exactly two tetrahedra, whose opposite vertices lie on
  opposite sides of it; the faces used once form a closed, locally convex surface, so they are the convex hull's
  triangulated facets; on every interior face the opposite vertex is not strictly inside the other tetrahedron's
  circumsphere (local Delaunay on a proper tiling is global Delaunay); every unique point is used, and no dropped
  duplicate is.  The signs are computed in float64 with a static error bound, vectorised, and only uncertain ones
  are recomputed exactly, so the check scales to 10^6-point outputs.
- `delaunay(xyz)` is a sequential Bowyer-Watson with a symbolic infinite vertex and the device's perturbation
  (DESIGN.md §4), for fixtures of a few thousand points.  It returns the same canonical array as the device.

Conventions (csrc/dt_predicates.cuh states the same ones): orient3d(a, b, c, d) = det[b - a; c - a; d - a];
insphere > 0 is strictly inside the circumsphere of a positively oriented tetrahedron.  Exactly on the sphere, the
points are ranked lexicographically by (x, y, z) and the two largest-ranked of the five decide, from the largest
down: the query point itself means outside, else orient3d with the query in that point's place, when nonzero
(Devillers and Teillaud's perturbation, as CGAL implements it).  A point coplanar with a hull facet is tested
against the facet's circumcircle, perturbed the same way with the coplanar orientation of the (x, y), (y, z) or
(x, z) projection.
"""
import numpy as np

__all__ = ["unique_points", "delaunay", "canonical", "certificate", "orient3d", "insphere"]

SCALE = 149
INF = -1
_EPS = 2.0 ** -53
_O2D = 2.0 * (3.0 + 16.0 * _EPS) * _EPS
_O3D = 2.0 * (7.0 + 56.0 * _EPS) * _EPS
_ISP = 2.0 * (16.0 + 224.0 * _EPS) * _EPS


def _int(v):
    n, d = float(v).as_integer_ratio()
    return n * ((1 << SCALE) // d)


def _ints(xyz):
    return [tuple(_int(c) for c in row) for row in np.asarray(xyz, dtype=np.float64)]


def _sgn(v):
    return (v > 0) - (v < 0)


# ------------------------------------------------------------------------------ exact predicates on integers
def _orient3d_i(a, b, c, d):
    bx, by, bz = b[0] - a[0], b[1] - a[1], b[2] - a[2]
    cx, cy, cz = c[0] - a[0], c[1] - a[1], c[2] - a[2]
    dx, dy, dz = d[0] - a[0], d[1] - a[1], d[2] - a[2]
    return _sgn(bx * (cy * dz - cz * dy) - by * (cx * dz - cz * dx) + bz * (cx * dy - cy * dx))


def _insphere_i(a, b, c, d, e):
    rows = []
    for p in (a, b, c, d):
        x, y, z = p[0] - e[0], p[1] - e[1], p[2] - e[2]
        rows.append((x, y, z, x * x + y * y + z * z))
    # det[[p - e, |p - e|^2]] = det[[x y z w 1]] = -insphere
    return -_sgn(_det4(rows))


def _det3(m):
    return (m[0][0] * (m[1][1] * m[2][2] - m[1][2] * m[2][1]) - m[0][1] * (m[1][0] * m[2][2] - m[1][2] * m[2][0])
            + m[0][2] * (m[1][0] * m[2][1] - m[1][1] * m[2][0]))


def _det4(m):
    out = 0
    for c in range(4):
        minor = [[m[r][k] for k in range(4) if k != c] for r in range(1, 4)]
        out += (-1) ** c * m[0][c] * _det3(minor)
    return out


_PROJ = ((0, 1), (1, 2), (0, 2))


def _orient2d_i(a, b, c, k):
    u, v = _PROJ[k]
    return _sgn((a[u] - c[u]) * (b[v] - c[v]) - (a[v] - c[v]) * (b[u] - c[u]))


def _incircle_i(a, b, c, d, k):
    u, v = _PROJ[k]
    rows = []
    for p in (a, b, c):
        pu, pv = p[u] - d[u], p[v] - d[v]
        dx, dy, dz = p[0] - d[0], p[1] - d[1], p[2] - d[2]
        rows.append((pu, pv, dx * dx + dy * dy + dz * dz))
    return _sgn(_det3(rows))


def _coplanar_orient_i(a, b, c):
    for k in range(3):
        o = _orient2d_i(a, b, c, k)
        if o:
            return o
    return 0


def orient3d(a, b, c, d):
    """Exact sign of det[b - a; c - a; d - a] for float coordinate triples."""
    return _orient3d_i(*(_ints([a, b, c, d])))


def insphere(a, b, c, d, e):
    """Exact sign: > 0 when e is strictly inside the circumsphere of the positively oriented (a, b, c, d)."""
    return _insphere_i(*(_ints([a, b, c, d, e])))


class _Points:
    """Exact coordinates and lexicographic ranks of the unique points."""

    def __init__(self, xyz, ids):
        self.P = _ints(np.asarray(xyz, dtype=np.float64)[ids])
        x = np.asarray(xyz, dtype=np.float64)[ids] + 0.0
        order = np.lexsort((x[:, 2], x[:, 1], x[:, 0]))
        self.rank = np.empty(len(ids), dtype=np.int64)
        self.rank[order] = np.arange(len(ids))

    def orient(self, a, b, c, d):
        P = self.P
        return _orient3d_i(P[a], P[b], P[c], P[d])

    def insphere_perturbed(self, v, e):
        P = self.P
        s = _insphere_i(P[v[0]], P[v[1]], P[v[2]], P[v[3]], P[e])
        if s:
            return s
        pts = list(v) + [e]
        order = sorted(range(5), key=lambda i: self.rank[pts[i]])
        for i in (4, 3):
            w = order[i]
            if w == 4:
                return -1
            q = list(v)
            q[w] = e
            o = self.orient(*q)
            if o:
                return o
        return -1

    def incircle_perturbed(self, v, d):
        P = self.P
        a, b, c = (P[i] for i in v)
        for k in range(3):
            local = _orient2d_i(a, b, c, k)
            if local:
                break
        ic = _incircle_i(a, b, c, P[d], k)
        if ic:
            return ic * local
        pts = list(v) + [d]
        order = sorted(range(4), key=lambda i: self.rank[pts[i]])
        for i in (3, 2, 1):
            w = order[i]
            if w == 3:
                return -1
            q = [P[i] for i in v]
            q[w] = P[d]
            o = _coplanar_orient_i(*q)
            if o:
                return o * local
        return -1

    def conflict(self, t, p):
        """Whether p lies inside the perturbed circumsphere of tetrahedron t (or sees an infinite one's facet)."""
        if INF in t:
            k = t.index(INF)
            q = list(t)
            q[k] = p
            o = self.orient(*q)
            if o:
                return o > 0
            return self.incircle_perturbed([t[i] for i in range(4) if i != k], p) > 0
        return self.insphere_perturbed(t, p) > 0


# ------------------------------------------------------------------------------ duplicates and canonical order
def unique_points(xyz):
    """Indices of the points kept (the smallest index of every group of exact duplicates, -0 equal to +0),
    ascending."""
    x = np.asarray(xyz, dtype=np.float32).astype(np.float64) + 0.0
    order = np.lexsort((np.arange(len(x)), x[:, 2], x[:, 1], x[:, 0]))
    xs = x[order]
    first = np.ones(len(x), dtype=bool)
    first[1:] = np.any(xs[1:] != xs[:-1], axis=1)
    return np.sort(order[first])


def canonical(simplices):
    """Rows rotated by an even permutation so that the smallest id comes first and the second smallest second,
    then sorted lexicographically; int64."""
    s = np.asarray(simplices, dtype=np.int64).reshape(-1, 4)
    if len(s) == 0:
        return s.copy()
    # the even permutations that bring position i to the front
    front = np.array([[0, 1, 2, 3], [1, 0, 3, 2], [2, 3, 0, 1], [3, 2, 1, 0]])
    s = np.take_along_axis(s, front[np.argmin(s, axis=1)], axis=1)
    # a cyclic rotation of the last three brings the second smallest to position 1
    rot = np.array([[0, 1, 2, 3], [0, 2, 3, 1], [0, 3, 1, 2]])
    s = np.take_along_axis(s, rot[np.argmin(s[:, 1:], axis=1)], axis=1)
    return s[np.lexsort((s[:, 3], s[:, 2], s[:, 1], s[:, 0]))]


# ------------------------------------------------------------------------------ sequential Bowyer-Watson
def delaunay(xyz):
    """The perturbed Delaunay triangulation of the unique points of xyz, canonical (int64 [T, 4]).
    ValueError when fewer than 4 unique points are affinely independent."""
    ids = unique_points(xyz)
    pts = _Points(xyz, ids)
    m = len(ids)
    P = pts.P
    if m < 4:
        raise ValueError("fewer than 4 affinely independent points")
    i2 = next((i for i in range(2, m) if _coplanar_orient_i(P[0], P[1], P[i]) != 0), None)
    if i2 is None:
        raise ValueError("fewer than 4 affinely independent points")
    i3 = next((i for i in range(2, m) if pts.orient(0, 1, i2, i) != 0), None)
    if i3 is None:
        raise ValueError("fewer than 4 affinely independent points")
    first = [0, 1, i2, i3]
    if pts.orient(*first) < 0:
        first[0], first[1] = first[1], first[0]
    tets, adj, alive = [first], [[None] * 4], [True]
    for i in range(4):
        t = list(first)
        t[i] = INF
        o = [j for j in range(4) if j != i]
        t[o[0]], t[o[1]] = t[o[1]], t[o[0]]
        tets.append(t)
        adj.append([None] * 4)
        alive.append(True)
        adj[0][i] = (i + 1, i)
        adj[i + 1][i] = (0, i)
    for i in range(4):
        for j in range(4):
            if i != j:
                # inf_i and inf_j share the face holding INF and the two vertices other than first[i], first[j]
                adj[i + 1][tets[i + 1].index(first[j])] = (j + 1, tets[j + 1].index(first[i]))
    last = 0
    for p in range(m):
        if p in first:
            continue
        start = _walk(pts, tets, adj, last, p)
        cav, seen, bnd = [start], {start}, []
        k = 0
        while k < len(cav):
            t = cav[k]
            k += 1
            for f in range(4):
                nb, nf = adj[t][f]
                if nb in seen:
                    continue
                if pts.conflict(tets[nb], p):
                    seen.add(nb)
                    cav.append(nb)
                else:
                    bnd.append((t, f))
        faces = {}
        new = []
        for t, f in bnd:
            v = list(tets[t])
            v[f] = p
            nid = len(tets)
            tets.append(v)
            alive.append(True)
            a = [None] * 4
            nb, nf = adj[t][f]
            a[f] = (nb, nf)
            adj[nb][nf] = (nid, f)
            adj.append(a)
            new.append(nid)
            for g in range(4):
                if g != f:
                    key = frozenset(v[h] for h in range(4) if h != g)
                    if key in faces:
                        o, og = faces.pop(key)
                        adj[nid][g] = (o, og)
                        adj[o][og] = (nid, g)
                    else:
                        faces[key] = (nid, g)
        assert not faces, "Bowyer-Watson cavity is not a ball"
        for t in cav:
            alive[t] = False
        last = next(t for t in new if INF not in tets[t]) if any(INF not in tets[t] for t in new) else new[0]
    out = np.array([t for t, a in zip(tets, alive) if a and INF not in t], dtype=np.int64)
    return canonical(ids[out])


def _walk(pts, tets, adj, t, p, max_steps=10 ** 7):
    """A tetrahedron in conflict with p: visibility walk from t (the one containing p, or an infinite one whose
    facet p sees)."""
    for step in range(max_steps):
        v = tets[t]
        if INF in v:
            k = v.index(INF)
            if pts.conflict(v, p):
                return t
            t = adj[t][k][0]
            continue
        moved = False
        for s in range(4):
            i = (s + p + step) & 3
            q = list(v)
            q[i] = p
            if pts.orient(*q) < 0:
                t = adj[t][i][0]
                moved = True
                break
        if not moved:
            return t
    raise RuntimeError("point location did not terminate")


# ------------------------------------------------------------------------------ certificate
def _orient_f(A, B, C, D):
    """Filtered orient3d of row-aligned float64 arrays [m, 3]: the sign where certain, 0 where not."""
    ad, bd, cd = A - D, B - D, C - D
    bxcy, cxby = bd[:, 0] * cd[:, 1], cd[:, 0] * bd[:, 1]
    cxay, axcy = cd[:, 0] * ad[:, 1], ad[:, 0] * cd[:, 1]
    axby, bxay = ad[:, 0] * bd[:, 1], bd[:, 0] * ad[:, 1]
    det = ad[:, 2] * (bxcy - cxby) + bd[:, 2] * (cxay - axcy) + cd[:, 2] * (axby - bxay)
    perm = ((np.abs(bxcy) + np.abs(cxby)) * np.abs(ad[:, 2]) + (np.abs(cxay) + np.abs(axcy)) * np.abs(bd[:, 2])
            + (np.abs(axby) + np.abs(bxay)) * np.abs(cd[:, 2]))
    bound = _O3D * perm
    return np.where(det > bound, -1, np.where(-det > bound, 1, 0))


def _insphere_f(A, B, C, D, E):
    a, b, c, d = A - E, B - E, C - E, D - E
    ab = a[:, 0] * b[:, 1] - b[:, 0] * a[:, 1]
    bc = b[:, 0] * c[:, 1] - c[:, 0] * b[:, 1]
    cd = c[:, 0] * d[:, 1] - d[:, 0] * c[:, 1]
    da = d[:, 0] * a[:, 1] - a[:, 0] * d[:, 1]
    ac = a[:, 0] * c[:, 1] - c[:, 0] * a[:, 1]
    bd = b[:, 0] * d[:, 1] - d[:, 0] * b[:, 1]
    abc = a[:, 2] * bc - b[:, 2] * ac + c[:, 2] * ab
    bcd = b[:, 2] * cd - c[:, 2] * bd + d[:, 2] * bc
    cda = c[:, 2] * da + d[:, 2] * ac + a[:, 2] * cd
    dab = d[:, 2] * ab + a[:, 2] * bd + b[:, 2] * da
    al, bl, cl, dl = ((v * v).sum(1) for v in (a, b, c, d))
    det = (dl * abc - cl * dab) + (bl * cda - al * bcd)

    def p2(u, v):
        return np.abs(u[:, 0] * v[:, 1]) + np.abs(v[:, 0] * u[:, 1])

    az, bz, cz, dz = (np.abs(v[:, 2]) for v in (a, b, c, d))
    pab, pbc, pcd, pda, pac, pbd = p2(a, b), p2(b, c), p2(c, d), p2(d, a), p2(a, c), p2(b, d)
    perm = ((pcd * bz + pbd * cz + pbc * dz) * al + (pda * cz + pac * dz + pcd * az) * bl
            + (pab * dz + pbd * az + pda * bz) * cl + (pbc * az + pac * bz + pab * cz) * dl)
    bound = _ISP * perm
    return np.where(det > bound, -1, np.where(-det > bound, 1, 0))


def _exact_fill(sign, fn, *cols):
    """Recomputes the uncertain (0) entries of a filtered sign exactly."""
    for i in np.flatnonzero(sign == 0):
        sign[i] = fn(*(_ints([c[i]])[0] for c in cols))
    return sign


def certificate(xyz, simplices, return_reason=False):
    """True when simplices (int [T, 4]) is the Delaunay triangulation of the unique points of xyz (see the module
    docstring for what is checked).  With return_reason, (ok, reason)."""
    def fail(why):
        return (False, why) if return_reason else False

    X = np.asarray(xyz, dtype=np.float32).astype(np.float64)
    S = np.asarray(simplices, dtype=np.int64).reshape(-1, 4)
    n = len(X)
    if len(S) == 0:
        return fail("no tetrahedron")
    if S.min() < 0 or S.max() >= n:
        return fail("an id out of range")
    keep = unique_points(X)
    used = np.zeros(n, dtype=bool)
    used[S.ravel()] = True
    kept = np.zeros(n, dtype=bool)
    kept[keep] = True
    if np.any(used & ~kept):
        return fail("a dropped duplicate is used")
    if not np.all(used[keep]):
        return fail("a unique point is not used")
    A, B, C, D = (X[S[:, i]] for i in range(4))
    o = _exact_fill(_orient_f(A, B, C, D), _orient3d_i, A, B, C, D)
    if np.any(o <= 0):
        return fail("a tetrahedron is not positively oriented")
    # faces: face i of a tetrahedron leaves out vertex i
    T = len(S)
    F = np.concatenate([np.delete(S, i, axis=1) for i in range(4)])
    opp = np.concatenate([S[:, i] for i in range(4)])
    tet = np.tile(np.arange(T), 4)
    key = np.sort(F, axis=1)
    order = np.lexsort((key[:, 2], key[:, 1], key[:, 0]))
    ks = key[order]
    new = np.ones(len(ks), dtype=bool)
    new[1:] = np.any(ks[1:] != ks[:-1], axis=1)
    start = np.flatnonzero(new)
    count = np.diff(np.append(start, len(ks)))
    if np.any(count > 2):
        return fail("a face is shared by more than two tetrahedra")
    two = start[count == 2]
    f1, f2 = order[two], order[two + 1]
    K = ks[two]
    P0, P1, P2 = (X[K[:, i]] for i in range(3))
    s1 = _exact_fill(_orient_f(P0, P1, P2, X[opp[f1]]), _orient3d_i, P0, P1, P2, X[opp[f1]])
    s2 = _exact_fill(_orient_f(P0, P1, P2, X[opp[f2]]), _orient3d_i, P0, P1, P2, X[opp[f2]])
    if np.any(s1 * s2 >= 0):
        return fail("an interior face has both tetrahedra on one side")
    # local Delaunay: the opposite vertex of the second tetrahedron against the first one's circumsphere
    t1 = S[tet[f1]]
    Q = [X[t1[:, i]] for i in range(4)]
    E = X[opp[f2]]
    ins = _exact_fill(_insphere_f(*Q, E), _insphere_i, *Q, E)
    if np.any(ins > 0):
        return fail("an interior face is not locally Delaunay")
    # hull: the faces used once, oriented outward, form a closed locally convex surface
    one = order[start[count == 1]]
    if len(one) < 4:
        return fail("the boundary is not a closed surface")
    hf = F[one]
    ho = opp[one]
    # orient each hull face so that its tetrahedron's opposite vertex is on its negative side
    Hp = [X[hf[:, i]] for i in range(3)]
    so = _exact_fill(_orient_f(*Hp, X[ho]), _orient3d_i, *Hp, X[ho])
    hf = np.where((so > 0)[:, None], hf[:, [1, 0, 2]], hf)
    # directed edges: every edge of the hull must appear once in each direction
    e = np.concatenate([hf[:, [0, 1]], hf[:, [1, 2]], hf[:, [2, 0]]])
    third = np.concatenate([hf[:, 2], hf[:, 0], hf[:, 1]])
    fe = np.tile(np.arange(len(hf)), 3)
    ek = e[:, 0] * n + e[:, 1]
    rk = e[:, 1] * n + e[:, 0]
    if len(np.unique(ek)) != len(ek):
        return fail("the hull surface is not a manifold")
    pos = np.searchsorted(np.sort(ek), rk)
    srt = np.argsort(ek)
    if np.any(pos >= len(ek)) or np.any(np.sort(ek)[np.minimum(pos, len(ek) - 1)] != rk):
        return fail("the hull surface is not closed")
    mate = srt[pos]
    # local convexity: the far vertex of the neighbouring face is not strictly outside this face's plane
    G = [X[hf[fe, i]] for i in range(3)]
    far = X[third[mate]]
    cv = _exact_fill(_orient_f(*G, far), _orient3d_i, *G, far)
    if np.any(cv > 0):
        return fail("the hull surface is not convex")
    return (True, "ok") if return_reason else True
