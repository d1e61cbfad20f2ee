"""Constructed neighbour sets for the match stage (search, neighbour order, plane fit, gates).

Every query gets its own cluster of map points, 24 m from the next one, so that its five nearest map points are exactly the
set built for it.  Coordinates are multiples of a grid step (2^-6 m near the origin, 2^-5 m far from it, 2^-3 m for the wide
variants) and query-to-point offsets stay below 2 m: differences, squares and sums of squares are then exact in fp32 and a
tie is a tie whatever order the terms are added in.  The state is the identity, so the world point is the query bit for bit.

A family comes in a compact variant (the five neighbours inside a quarter metre: level 0 settles it) and a wide one (the
fifth beyond a metre: the ring search).  The families:
  tie          2, 3 or 5 equidistant neighbours with distinct x
  equal_x      equidistant pairs with equal x: mirror images about the query in y or z, and (a, b, c) / (a, c, b)
  duplicate    2, 3 or 5 copies of one map point
  collinear    five points on one line (rank 1), and the same with one coordinate one ulp off it
  rank2        five coplanar points in general position (rank 2 of the centred set, full rank of A)
and, near the origin only (their defining property is in absolute coordinates):
  origin_plane coplanar points on a plane through the origin (A n = -1 has no exact solution), and that plane one ulp off
  origin_line  points on a line through the origin
  zero_column  every x exactly 0
  equal_norms  rows (a, b, c), (b, c, a), (c, a, b), (d, d, d), (e, e, e): three equal column norms, tied pivots
and apart: nan_case (five copies of the origin), near_tie_cases (near-ties inside the comparator's 1e-10 window) and
adversarial_sets (sets for the fit alone).
"""
import itertools

import numpy as np

SPACING = 24.0
ORIGINS = {"origin": (0.0, 0.0, 0.0), "far_a": (2e5, -3e5, 50.0), "far_b": (4.3e5, 0.0, 0.0)}
FRAC = 0.3125                       # 10 / 32: the query's place in its cluster cell, on the grid at every origin


def grid_step(origin, wide):
    if wide:
        return 2.0 ** -3
    return 2.0 ** -6 if origin == "origin" else 2.0 ** -5


_R = np.arange(-16, 17)
_V = np.stack(np.meshgrid(_R, _R, _R, indexing="ij"), -1).reshape(-1, 3)
_N2 = (_V * _V).sum(1)
_BY_N2 = {int(n): _V[_N2 == n] for n in np.unique(_N2) if n <= 256}


def sphere(n2):
    """every integer vector with squared norm n2 (n2 <= 256)"""
    return _BY_N2.get(int(n2), np.zeros((0, 3), np.int64))


class Case:
    def __init__(self, family, query, points, ties=()):
        self.family = family
        self.query = np.asarray(query, np.float32)
        self.points = np.asarray(points, np.float32).reshape(-1, 3)
        self.ties = tuple(ties)      # pairs of indices into points that are equidistant with equal x


def _fill(rng, used_n2, k, lo, hi):
    """k vectors of pairwise distinct squared norms in [lo, hi], none in used_n2"""
    out = []
    cand = [n for n in range(lo, hi + 1) if n not in used_n2 and len(sphere(n)) > 0]
    for n in rng.choice(cand, size=k, replace=False):
        s = sphere(int(n))
        out.append(s[rng.integers(len(s))])
    return out


def _sets(rng, lo, hi):
    """(family, five integer vectors, tied equal-x pairs) at squared norms in [lo, hi]"""
    out = []
    rich = [n for n in range(lo, hi + 1) if len(np.unique(sphere(n)[:, 0])) >= 5]
    for m in (2, 3, 5):                                               # exact ties, distinct x
        for _ in range(6):
            n = int(rng.choice(rich))
            s = sphere(n)
            xs = rng.permutation(np.unique(s[:, 0]))[:m]
            tied = [s[s[:, 0] == x][rng.integers((s[:, 0] == x).sum())] for x in xs]
            v = tied + _fill(rng, {n}, 5 - m, lo, hi)
            out.append(("tie", v, ()))
    for kind in ("mirror_y", "mirror_z", "swap_yz", "two_pairs"):    # equidistant, equal x
        for _ in range(8):
            n = int(rng.choice(rich))
            s = sphere(n)
            if kind == "swap_yz":
                s = s[s[:, 1] != s[:, 2]]
            else:
                s = s[(s[:, 1] != 0) & (s[:, 2] != 0)]
            a = s[rng.integers(len(s))]
            b = a * (1, -1, 1) if kind in ("mirror_y", "two_pairs") else (a * (1, 1, -1) if kind == "mirror_z" else a[[0, 2, 1]])
            v = [a, b]
            pairs = [(0, 1)]
            if kind == "two_pairs":
                n2 = int(rng.choice([r for r in rich if r != n]))
                s2 = sphere(n2)
                s2 = s2[(s2[:, 2] != 0)]
                c = s2[rng.integers(len(s2))]
                v += [c, c * (1, 1, -1)]
                pairs.append((2, 3))
                v += _fill(rng, {n, n2}, 1, lo, hi)
            else:
                v += _fill(rng, {n}, 3, lo, hi)
            out.append(("equal_x", v, tuple(pairs)))
    for m in (2, 3, 5):                                               # duplicates
        for _ in range(4):
            a = _fill(rng, set(), 1, lo, hi)[0]
            v = [a] * m + _fill(rng, {int((a * a).sum())}, 5 - m, lo, hi)
            out.append(("duplicate", v, ()))
    for _ in range(6):                                                # collinear (rank 1)
        d = rng.integers(-3, 4, 3)
        while not d.any():
            d = rng.integers(-3, 4, 3)
        a = rng.integers(-2, 3, 3)
        v = [a + t * d for t in (1, 2, 3, -1, -2)]
        out.append(("collinear", v, ()))
    for _ in range(6):                                                # five coplanar points
        e1, e2 = rng.integers(-3, 4, 3), rng.integers(-3, 4, 3)
        c = rng.integers(-2, 3, 3)
        v = [c + i * e1 + j * e2 for i, j in ((1, 0), (0, 1), (2, 1), (-1, 2), (1, -2))]
        out.append(("rank2", v, ()))
    return out


def _lattice_query(origin, slot, width=8):
    o = np.asarray(ORIGINS[origin], np.float64)
    i, j = slot % width, slot // width
    return o + (SPACING * i + FRAC, SPACING * (j + 1) + FRAC, FRAC)


def _nudge_one(v, rng):
    """one coordinate of one point moved by one fp32 ulp"""
    v = np.array(v, np.float32)
    r, c = rng.integers(len(v)), rng.integers(3)
    v[r, c] = np.nextafter(v[r, c], np.float32(np.inf))
    return v


def origin_specials():
    """the sets whose property is in absolute coordinates, each at its own place near the origin"""
    u = 2.0 ** -6
    rng = np.random.default_rng(3)

    def plane(cx, cy):                     # on x + y + z = 0
        return np.array([(cx + a * u, cy + b * u, -(cx + cy) - (a + b) * u) for a, b in ((3, 1), (-2, 5), (4, -3), (-5, -1), (1, 6))])

    def line(cx, cy):                      # on t (cx, cy, 0)
        return np.array([(cx * (1 + t * u), cy * (1 + t * u), 0.0) for t in (1, -2, 3, -1, 2)])

    out = [Case("origin_plane", (8.0, -8.0, u), plane(8.0, -8.0)),
           Case("origin_plane_ulp", (16.0, -16.0, u), _nudge_one(plane(16.0, -16.0), rng)),
           Case("origin_line", (8.0, -16.0, u * 3), line(8.0, -16.0)),
           Case("origin_line_ulp", (16.0, -32.0, u * 3), _nudge_one(line(16.0, -32.0), rng)),
           Case("zero_column", (u * 4, -8.0, 8.0), [(0.0, -8 + b * u, 8 + c * u) for b, c in ((1, 2), (-3, 1), (4, -2), (-1, -5), (6, 3))])]
    a, b, c, d, e = (-8 + k * u for k in (1, 3, -2, 5, -4))
    out.append(Case("equal_norms", (-8.0, -8.0, -8.0), [(a, b, c), (b, c, a), (c, a, b), (d, d, d), (e, e, e)]))
    return out


def nan_case():
    """five copies of the origin, a map of their own: the fit divides by a zero pivot and returns a NaN plane, which is_plane
    accepts (|NaN| > threshold is false); kept out of the other maps, whose normal equations it would make NaN"""
    return Case("origin_dup", (2.0 ** -3, 2.0 ** -4, 2.0 ** -5), np.zeros((5, 3)))


def build(origin="origin", wide=False, seed=0):
    """(map points, queries, cases) for one origin and variant"""
    rng = np.random.default_rng(1000 * seed + (7 if wide else 0) + list(ORIGINS).index(origin))
    step = grid_step(origin, wide)
    lo, hi = (64, 196) if wide else (16, 256)          # squared norms in grid units: wide 1.0 .. 1.75 m, compact <= 0.25 m (near)
    cases = []
    for slot, (fam, v, pairs) in enumerate(_sets(rng, lo, hi)):
        q = _lattice_query(origin, slot)
        pts = q + np.asarray(v, np.float64) * step
        assert (pts.astype(np.float32) == pts).all() and (q.astype(np.float32) == q).all()   # on the grid: exact in fp32
        c = Case(fam, q, pts, pairs)
        if fam == "collinear" and slot % 2:
            c = Case("collinear_ulp", q, _nudge_one(pts, rng))
        cases.append(c)
    if origin == "origin" and not wide:
        cases += origin_specials()
    pts = np.concatenate([c.points for c in cases]).astype(np.float32)
    qs = np.stack([c.query for c in cases]).astype(np.float32)
    return pts, qs, cases


def point_ids(cases):
    """map point ids (insertion order) of each case's points"""
    out, k = [], 0
    for c in cases:
        out.append(np.arange(k, k + len(c.points)))
        k += len(c.points)
    return out


def sq_dist32(q, p):
    """KD_TREE::calc_dist in fp32, ((dx^2 + dy^2) + dz^2), unfused"""
    d = np.asarray(q, np.float32) - np.asarray(p, np.float32)
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def expected_order(case, ids):
    """the five neighbours in the product's order: ascending (distance, x, y, z, id) — exact ties only in these sets"""
    d = sq_dist32(case.query, case.points)
    keys = [(float(d[i]), float(case.points[i, 0]), float(case.points[i, 1]), float(case.points[i, 2]), int(ids[i]))
            for i in range(len(ids))]
    order = sorted(range(len(ids)), key=lambda i: keys[i])[:5]
    return np.asarray(ids)[order], d[order]


def halo_positions(dump, q, k, ids):
    """positions of map point ids in the halo bucket of q's home voxel (map_ref layout), -1 where absent"""
    import map_ref
    lay = dump.layout()
    key = map_ref.pack(map_ref.voxels(map_ref.cells(np.asarray(q, np.float32)[None]), k)[0])[0]
    s = int(np.searchsorted(lay.slot_keys, key))
    if s >= len(lay.slot_keys) or lay.slot_keys[s] != key:
        return np.full(len(ids), -1)
    start = int(lay.halo_counts[:s].sum())
    bucket = lay.halo_flat[start:start + int(lay.halo_counts[s]), 3].astype(np.int64)
    return np.array([int(np.nonzero(bucket == i)[0][0]) if (bucket == i).any() else -1 for i in ids])


def lane_order(pa, pb, g):
    """True when position pa comes out of a g-lane scan before pb at equal distance: lowest lane first, then earlier"""
    return (pa % g, pa) < (pb % g, pb)


def permutations5():
    return list(itertools.permutations(range(5)))


def near_tie_cases(n=400, seed=5):
    """Near-ties inside PointType_CMP's 1e-10 window (ikd_Tree.h:109-115), neighbours within 1 cm, clusters 0.5 m apart within
    4 m of the origin (a coordinate ulp <= 2^-22 m, so neighbouring fp32 squared distances are reachable).  Per query: three
    clear neighbours at 2, 3 and 4 mm, then three points a < b < c in raw fp32 squared distance with c - a < 1e-10 and
    x(a) > x(c): under the comparator a ranks above c, so a heap whose top is a rejects b (ikd_Tree.cpp:1087: dist < top),
    though the exact 5-NN holds b and not c."""
    rng = np.random.default_rng(seed)
    cases = []
    side = int(np.ceil(n ** (1 / 3)))
    for s in range(n):
        cell = np.array([s % side, (s // side) % side, s // (side * side)], np.float64)
        q = (cell * 0.5 - 3.5 + rng.uniform(0.05, 0.1, 3)).astype(np.float32)
        near = []
        for r in (0.002, 0.003, 0.004):
            u = rng.normal(size=3)
            near.append(q + (r * u / np.linalg.norm(u)).astype(np.float32))
        u = rng.normal(size=(4000, 3))
        pool = (q + (0.006 * u / np.linalg.norm(u, axis=1, keepdims=True))).astype(np.float32)
        d = sq_dist32(q, pool)
        o = np.argsort(d, kind="stable")
        pool, d = pool[o], d[o]
        pick = None
        for i in range(len(d) - 2):
            j = i + 1
            while j < len(d) and d[j] == d[i]:
                j += 1
            k = j + 1
            while k < len(d) and d[k] == d[j]:
                k += 1
            if k < len(d) and np.float32(d[k] - d[i]) < 1e-10 and d[i] < d[j] < d[k] and pool[i, 0] > pool[k, 0]:
                pick = (i, j, k)
                break
        if pick is None:
            continue
        pts = np.array(near + [pool[pick[0]], pool[pick[1]], pool[pick[2]]], np.float32)
        cases.append(Case("near_tie", q, pts[rng.permutation(6)]))
    return cases


def adversarial_sets(n=100000, seed=9):
    """n five-point sets for the fit alone (q: n x 5 x 3, g: n x 3, ids: n x 5), in random row order: near-collinear sets one to
    64 ulps off their line, tied pivots (cyclic rows: equal column norms), equidistant and duplicate rows (the tie order),
    near the origin and at 2e5 m"""
    rng = np.random.default_rng(seed)
    kind = rng.integers(0, 4, n)
    off = np.where(rng.random(n)[:, None] < 0.25, np.array([2e5, -3e5, 50.0]), 0.0) + rng.uniform(-30, 30, (n, 3))
    g = off.astype(np.float32)
    q = np.zeros((n, 5, 3), np.float64)
    t = rng.uniform(-1, 1, (n, 5, 1))
    dirn = rng.normal(size=(n, 1, 3))
    q[kind == 0] = (t * dirn)[kind == 0]                                            # collinear
    abc = rng.uniform(-1, 1, (n, 3))
    cyc = np.stack([abc, abc[:, [1, 2, 0]], abc[:, [2, 0, 1]], np.repeat(abc[:, :1], 3, 1), np.repeat(abc[:, 1:2], 3, 1)], 1)
    q[kind == 1] = cyc[kind == 1]                                                   # equal column norms
    e1, e2 = rng.normal(size=(n, 1, 3)), rng.normal(size=(n, 1, 3))
    q[kind >= 2] = (rng.uniform(-1, 1, (n, 5, 1)) * e1 + rng.uniform(-1, 1, (n, 5, 1)) * e2)[kind >= 2]   # planar
    m = kind == 3                                                                  # mirror pairs / duplicates about g
    q[m, 1] = q[m, 0] * np.array([1.0, -1.0, 1.0])
    q[m, 3] = q[m, 2]
    q = (q + g[:, None, :].astype(np.float64)).astype(np.float32)
    k = rng.integers(1, 65, n)                                                     # one coordinate k ulps off
    r, c = rng.integers(0, 5, n), rng.integers(0, 3, n)
    v = q[np.arange(n), r, c]
    q[np.arange(n), r, c] = v + (k * np.spacing(np.abs(v))).astype(np.float32) * np.where(kind == 0, 1, 0)
    perm = np.argsort(rng.random((n, 5)), 1)
    q = np.take_along_axis(q, perm[:, :, None], 1)
    ids = np.take_along_axis(np.tile(np.arange(5, dtype=np.int32), (n, 1)) + 5 * np.arange(n, dtype=np.int32)[:, None], perm, 1)
    return q, g, ids
