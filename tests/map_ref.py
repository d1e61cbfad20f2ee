"""Mapper::add on the voxel map, restated in numpy, and an independent checker of the map's layout.

The restatement (`MapRef`) follows DESIGN.md §3 and the reference's text (`ikd_Tree.cpp:478-573` Add_Points with the
downsample rule, `:1246-1287` Search_by_range); it calls no product code.  Every fp32 operation is a numpy float32 operation,
rounded on its own (no FMA), as `lv_hd.h` does on the device.

  cell      floor(fl(v / ds)), ds = 0.2 (`ikd_Tree.cpp:491`)
  voxel     floor(cell / k) + 2^20, clamped to 21 bits; k = 1, 2, 3 (voxel 0.2 / 0.4 / 0.6)
  build     (downsample 0, or an add that builds an empty map) every storable point is appended; within a voxel in ascending
            cell index, then input order (the order of the radix-sorted run)
  add       per touched cell, in ascending cell index inside its voxel: the old points of the cell are the voxel's own points
            inside the cell's box [fl(c ds), fl(c ds) + ds) (Search_by_range's test, :1262); distances to the box centre as
            :497-502 compute them; the first strict minimum among old points, a new point beats an old one at equal
            distance, the later of two equal new points wins; a single old point that wins, or a winning new point equal to
            the single old one, changes nothing; otherwise the cell's old points go and the winner is appended
  ids       id_base + index in the add; id_base counts every submitted point, stored or not

What the ikd-Tree does differently is confined to `flagged` cells: where a point's index cell floor(q / ds) and the boxes
that contain it disagree, the tree's box test and the map's per-voxel cell test can pick different points.

Points whose voxel coordinate clamps (beyond +-209 715 m at voxel 0.2) are outside the restatement: `MapRef.clamped` counts
them, and a test that compares content asserts it is 0.  The layout checker (`check_layout`) needs no restatement and holds
at clamped keys too.
"""
import numpy as np

DS = np.float32(0.2)
KEY_BIAS, KEY_MAX = 1 << 20, 0x1FFFFF
EMPTY = 0xFFFFFFFF
FINITE_BOUND = np.float32(1e9)                   # map_point_key: |x|, |y|, |z| < 1e9 or the point is not stored
# device counter words (lv_voxel_map.h MapCounters)
CTR_ARENA_TOP, CTR_POINTS, CTR_TOUCHED, CTR_DIRTY, CTR_ERROR, CTR_SLOTS_USED, CTR_GATHER, CTR_BLOCKS_USED = range(8)
ARENA_FIRST = 16                                 # position 0 .. 15 of the arena is never handed out
BLOCK_MULT = np.uint32(0x9E3779B1)

# 27 neighbour offsets by neighbour number nb (nb % 3 - 1, nb / 3 % 3 - 1, nb / 9 - 1) and the halo lane order
NB_OFF = np.array([[nb % 3 - 1, (nb // 3) % 3 - 1, nb // 9 - 1] for nb in range(27)], np.int64)
LANE_NB = np.array([13] + list(range(13)) + list(range(14, 27)), np.int64)


# ---- geometry -------------------------------------------------------------------------------------------------------
def cells(xyz, ds=DS):
    """floor(fl(v / ds)) per coordinate, int64"""
    return np.floor(np.asarray(xyz, np.float32) / np.float32(ds)).astype(np.int64)


def voxels(c, k):
    """biased voxel coordinates of cells c and whether each coordinate clamped"""
    v = np.floor_divide(c, k) + KEY_BIAS
    return np.clip(v, 0, KEY_MAX), (v < 0) | (v > KEY_MAX)


def pack(b):
    b = np.asarray(b, np.uint64)
    return b[..., 0] | (b[..., 1] << np.uint64(21)) | (b[..., 2] << np.uint64(42))


def unpack(key):
    key = np.asarray(key, np.uint64)
    m = np.uint64(0x1FFFFF)
    return np.stack([key & m, (key >> np.uint64(21)) & m, (key >> np.uint64(42)) & m], -1).astype(np.int64)


def cell_lo(c, ds=DS):
    return c.astype(np.float32) * np.float32(ds)


def box_cell(q, ds=DS):
    """the cell whose box [fl(c ds), fl(c ds) + ds) holds q, looked for next to floor(q / ds) (the index cell)"""
    q = np.asarray(q, np.float32)
    c = cells(q, ds)
    lo = cell_lo(c, ds)
    below = q < lo
    above = ~below & ~(q < lo + np.float32(ds))
    return c - below + above


def centre_dist(q, c, ds=DS):
    """squared fp32 distance of q to the centre of cell c: vertex_min + (vertex_max - vertex_min) / 2.0 (:497-499, in double,
    stored as float), then calc_dist (:1682-1686)"""
    lo = cell_lo(c, ds)
    hi = lo + np.float32(ds)
    mid = (lo.astype(np.float64) + (hi - lo).astype(np.float64) / 2.0).astype(np.float32)
    d = np.asarray(q, np.float32) - mid
    return (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]


def storable(xyz):
    return (np.abs(np.asarray(xyz, np.float32)) < FINITE_BOUND).all(1)


def voxel_hash(key):
    """voxel_hash in uint32 arithmetic"""
    key = np.asarray(key, np.uint64)
    m = np.uint64(0x1FFFFF)
    x = (key & m).astype(np.uint32)
    y = ((key >> np.uint64(21)) & m).astype(np.uint32)
    z = ((key >> np.uint64(42)) & m).astype(np.uint32)
    with np.errstate(over="ignore"):
        h = (x * np.uint32(73856093)) ^ (y * np.uint32(19349663)) ^ (z * np.uint32(83492791))
        h ^= h >> np.uint32(15)
        h *= np.uint32(0x2C1B3C6D)
        h ^= h >> np.uint32(12)
    return h


def block_home(key):
    with np.errstate(over="ignore"):
        return voxel_hash(key) * BLOCK_MULT


# ---- flat extents ----------------------------------------------------------------------------------------------------
def _gather_index(starts, counts):
    """indices starts[i] + 0 .. counts[i]-1, concatenated"""
    starts, counts = np.asarray(starts, np.int64), np.asarray(counts, np.int64)
    total = int(counts.sum())
    if total == 0:
        return np.zeros(0, np.int64)
    off = np.cumsum(counts) - counts
    return np.repeat(starts - off, counts) + np.arange(total)


def _lookup(sorted_keys, keys):
    """position of each key in sorted_keys, -1 where absent"""
    pos = np.searchsorted(sorted_keys, keys)
    pos = np.minimum(pos, max(len(sorted_keys) - 1, 0))
    hit = (len(sorted_keys) > 0) & (sorted_keys[pos] == keys) if len(sorted_keys) else np.zeros(len(keys), bool)
    return np.where(hit, pos, -1)


def neighbour_keys(keys):
    """(n, 27) keys of the 27 neighbours in halo lane order, and whether each lies inside the key range"""
    b = unpack(keys)[:, None, :] + NB_OFF[LANE_NB][None, :, :]
    ok = ((b >= 0) & (b <= KEY_MAX)).all(-1)
    return pack(np.clip(b, 0, KEY_MAX)), ok


def halo_of(slot_keys, own_keys, own_counts, own_flat):
    """each slot's bucket: the own extents of its 27 neighbours in lane order (self first).  own_keys sorted; own_flat holds
    the extents one after another in that order.  Returns (counts per slot, the buckets one after another)"""
    own_off = np.cumsum(own_counts) - own_counts
    nk, ok = neighbour_keys(slot_keys)
    pos = _lookup(own_keys, nk.ravel()).reshape(nk.shape)
    pos[~ok] = -1
    cnt = np.where(pos >= 0, own_counts[np.maximum(pos, 0)], 0)
    st = np.where(pos >= 0, own_off[np.maximum(pos, 0)], 0)
    return cnt.sum(1), own_flat[_gather_index(st.ravel(), cnt.ravel())]


def blocks_of(own_keys):
    """sorted block keys and their 64-bit occupancy masks for the occupied voxels own_keys"""
    b = unpack(own_keys)
    bk = pack(b >> 2)
    bit = np.uint64(1) << ((b[:, 0] & 3) | ((b[:, 1] & 3) << 2) | ((b[:, 2] & 3) << 4)).astype(np.uint64)
    order = np.argsort(bk, kind="stable")
    bk, bit = bk[order], bit[order]
    keys, first = np.unique(bk, return_index=True)
    return keys, np.bitwise_or.reduceat(bit, first) if len(keys) else np.zeros(0, np.uint64)


def dilate(own_keys):
    nk, ok = neighbour_keys(own_keys)
    return np.unique(nk[ok])


class Layout:
    """a map's layout by voxel key, independent of table positions and arena offsets.  Points are uint32 (x, y, z, id) bits."""

    def __init__(self, slot_keys, own_keys, own_counts, own_flat, halo_counts, halo_flat, block_keys, block_masks, points,
                 slots_used, blocks_used, touched, dirty):
        self.slot_keys, self.own_keys, self.own_counts, self.own_flat = slot_keys, own_keys, own_counts, own_flat
        self.halo_counts, self.halo_flat = halo_counts, halo_flat
        self.block_keys, self.block_masks = block_keys, block_masks
        self.points, self.slots_used, self.blocks_used = int(points), int(slots_used), int(blocks_used)
        self.touched, self.dirty = touched, dirty            # sorted voxel keys of the last add's lists

    FIELDS = ("slot_keys", "own_keys", "own_counts", "own_flat", "halo_counts", "halo_flat", "block_keys", "block_masks",
              "points", "slots_used", "blocks_used", "touched", "dirty")

    def diff(self, other, lists=True):
        """names of the fields that differ (empty: equal bit for bit); lists=False leaves out the last add's lists"""
        out = []
        for f in self.FIELDS if lists else self.FIELDS[:-2]:
            a, b = getattr(self, f), getattr(other, f)
            if isinstance(a, int):
                if a != b:
                    out.append("%s %d != %d" % (f, a, b))
            elif a.shape != b.shape or not np.array_equal(a, b):
                out.append("%s %s != %s" % (f, a.shape, b.shape))
        return out

    def points_xyz(self):
        return self.own_flat[:, :3].view(np.float32)

    def ids(self):
        return self.own_flat[:, 3]


# ---- the restatement -------------------------------------------------------------------------------------------------
class MapRef:
    def __init__(self, k, ds=DS):
        self.k, self.ds = int(k), np.float32(ds)
        self.xyz = np.zeros((0, 3), np.float32)
        self.ids = np.zeros(0, np.uint32)
        self.vb = np.zeros((0, 3), np.int64)       # biased voxel coordinates
        self.key = np.zeros(0, np.uint64)
        self.ord = np.zeros(0, np.int64)           # own-extent order within a voxel
        self.next_ord = 0
        self.next_id = 0
        self.clamped = 0                           # storable points whose voxel coordinate clamped
        self.flagged = np.zeros((0, 3), np.int64)  # cells where box membership and index membership disagree
        self.cells_seen = np.zeros((0, 3), np.int64)
        self.touched = np.zeros(0, np.uint64)
        self.merge_paths = set()                   # "cached" / "uncached": which map_merge_run path each voxel run takes

    def clear(self):
        self.__init__(self.k, self.ds)

    def size(self):
        return len(self.ids)

    # -- flagged cells --
    def _flag(self, q):
        ds = self.ds
        ic = cells(q, ds)
        cand = ic[:, :, None] + np.array([-1, 0, 1])[None, None, :]           # (n, 3 axes, 3 candidates)
        lo = cell_lo(cand, ds)
        inbox = (lo <= q[:, :, None]) & (q[:, :, None] < lo + ds)
        alone = inbox[:, :, 1] & ~inbox[:, :, 0] & ~inbox[:, :, 2]             # S = {I} along this axis
        bad = ~alone.all(1)
        self.cells_seen = np.unique(np.concatenate([self.cells_seen, ic]), axis=0)
        if not bad.any():
            return
        # per axis: the boxes holding q, its index cell and the box cell_coord_old files it under (a gap between two boxes)
        bc = box_cell(q[bad], ds)
        sel = inbox[bad].copy()
        sel[:, :, 1] = True
        sel |= (bc[:, :, None] == cand[bad])
        out = []
        for a in range(3):
            for b in range(3):
                for c in range(3):
                    m = sel[:, 0, a] & sel[:, 1, b] & sel[:, 2, c]
                    cb = cand[bad]
                    out.append(np.stack([cb[m, 0, a], cb[m, 1, b], cb[m, 2, c]], 1))
        self.flagged = np.unique(np.concatenate([self.flagged] + out), axis=0)

    # -- one add --
    def add(self, xyz, downsample=True, count=None, min_points=0, build_if_empty=False):
        """Mapper::add of xyz.  count (a device count): clamped to len(xyz), none below max(min_points, 1); build_if_empty:
        an add that finds the map without points builds it"""
        xyz = np.ascontiguousarray(xyz, np.float32).reshape(-1, 3)
        n = len(xyz)
        if count is not None:
            n = int(min(max(count, 0), n))
            if n < max(min_points, 1):
                n = 0
            if build_if_empty and self.size() == 0:
                downsample = False
        xyz = xyz[:n]
        id_base = self.next_id
        self.next_id += n
        idx = np.nonzero(storable(xyz))[0]
        p = xyz[idx]
        k = self.k
        c = cells(p, self.ds)
        vb, cl = voxels(c, k)
        self.clamped += int(cl.any(1).sum())
        self._flag(p)
        key = pack(vb)
        loc = np.clip(c - (vb - KEY_BIAS) * k, 0, k - 1)
        li = loc[:, 0] + k * (loc[:, 1] + k * loc[:, 2])
        order = np.lexsort((idx, li, key))
        idx, p, c, vb, key, li = idx[order], p[order], c[order], vb[order], key[order], li[order]
        ids = (np.uint32(id_base) + idx.astype(np.uint32)).astype(np.uint32)
        if not downsample:
            self._append(p, ids, vb, key)
            self.touched = np.unique(key)
            self._note_paths(key, None, downsample)
            return
        # groups: one per (voxel, cell), the cell read from its first point
        new_g = np.ones(len(key), bool)
        new_g[1:] = (key[1:] != key[:-1]) | (li[1:] != li[:-1])
        gstart = np.nonzero(new_g)[0]
        gid = np.cumsum(new_g) - 1
        gkey, gcell = key[gstart], c[gstart]
        gend = np.append(gstart[1:], len(key))
        first_of_voxel = np.ones(len(gkey), bool)
        first_of_voxel[1:] = gkey[1:] != gkey[:-1]
        vstart = np.maximum.accumulate(np.where(first_of_voxel, np.arange(len(gkey)), 0))
        rank = np.arange(len(gkey)) - vstart
        self._note_paths(key, gkey, downsample)
        # new points: the last one at the group's minimum distance
        d_new = centre_dist(p, gcell[gid], self.ds)
        m_new = np.minimum.reduceat(d_new, gstart) if len(gstart) else np.zeros(0, np.float32)
        at_min = np.where(d_new == m_new[gid], np.arange(len(d_new)), -1)
        best_new = np.maximum.reduceat(at_min, gstart) if len(gstart) else np.zeros(0, np.int64)
        touched = []
        for r in range(int(rank.max()) + 1 if len(rank) else 0):
            g = np.nonzero(rank == r)[0]                                       # at most one group per voxel
            # old points of each group: own points of its voxel in its cell's box
            bc = box_cell(self.xyz, self.ds)
            okey = self.key
            gk = gkey[g]
            vpos = _lookup(gk, okey)                                           # gk is sorted: one group per voxel
            hit = vpos >= 0
            hit[hit] = (bc[hit] == gcell[g[vpos[hit]]]).all(1)
            ho = np.nonzero(hit)[0]
            hg = vpos[ho]                                                      # group (index into g) of each old point
            d_old = centre_dist(self.xyz[ho], gcell[g[hg]], self.ds)
            n_old = np.bincount(hg, minlength=len(g))
            o = np.lexsort((self.ord[ho], d_old, hg))                          # first strict minimum: earliest among equals
            first = np.ones(len(o), bool)
            first[1:] = hg[o][1:] != hg[o][:-1]
            best_old = np.full(len(g), -1, np.int64)
            best_old_d = np.full(len(g), np.inf, np.float32)
            best_old[hg[o][first]] = ho[o][first]
            best_old_d[hg[o][first]] = d_old[o][first]
            bn = best_new[g]
            take_new = ~(best_old_d < m_new[g])                                # no old point, or not strictly closer
            same = take_new & (n_old == 1)
            same[same] = (self.xyz[best_old[same]] == p[bn[same]]).all(1)
            change = (take_new | (n_old > 1)) & ~same
            if not change.any():
                continue
            gone = np.zeros(len(self.ids), bool)
            gone[ho[change[hg]]] = True
            ch = np.nonzero(change)[0]
            wn = ch[take_new[ch]]
            wo = ch[~take_new[ch]]
            # winners, in group order (one per voxel: their relative order does not matter)
            w_xyz = np.concatenate([p[bn[wn]], self.xyz[best_old[wo]]])
            w_ids = np.concatenate([ids[bn[wn]], self.ids[best_old[wo]]])
            w_vb = np.concatenate([vb[bn[wn]], self.vb[best_old[wo]]])
            w_key = np.concatenate([gkey[g[wn]], self.key[best_old[wo]]])
            keep = ~gone
            self.xyz, self.ids, self.vb, self.key, self.ord = (a[keep] for a in (self.xyz, self.ids, self.vb, self.key, self.ord))
            self._append(w_xyz, w_ids, w_vb, w_key)
            touched.append(gkey[g[ch]])
        self.touched = np.unique(np.concatenate(touched)) if touched else np.zeros(0, np.uint64)

    def _append(self, xyz, ids, vb, key):
        m = len(ids)
        self.xyz = np.concatenate([self.xyz, xyz])
        self.ids = np.concatenate([self.ids, ids])
        self.vb = np.concatenate([self.vb, vb])
        self.key = np.concatenate([self.key, key])
        self.ord = np.concatenate([self.ord, self.next_ord + np.arange(m)])
        self.next_ord += m

    def _note_paths(self, key, gkey, downsample):
        """map_merge_run caches the cell of every own point when the voxel's points plus one per group fit 48"""
        if not downsample or len(key) == 0:
            return
        vk, groups = np.unique(gkey, return_counts=True)
        own_k, own_n = np.unique(self.key, return_counts=True)
        pos = _lookup(own_k, vk)
        cnt = np.where(pos >= 0, own_n[np.maximum(pos, 0)], 0)
        fits = cnt + groups <= 48
        if fits.any():
            self.merge_paths.add("cached")
        if (~fits).any():
            self.merge_paths.add("uncached")

    # -- derived layout --
    def layout(self):
        order = np.lexsort((self.ord, self.key))
        key = self.key[order]
        flat = np.concatenate([self.xyz[order].view(np.uint32), self.ids[order][:, None]], 1)
        own_keys, own_counts = np.unique(key, return_counts=True)
        slot_keys = dilate(own_keys) if len(own_keys) else np.zeros(0, np.uint64)
        hc, hf = halo_of(slot_keys, own_keys, own_counts, flat)
        bk, bm = blocks_of(own_keys) if len(own_keys) else (np.zeros(0, np.uint64), np.zeros(0, np.uint64))
        dirty = np.unique(self._dirty()) if len(self.touched) else np.zeros(0, np.uint64)
        return Layout(slot_keys, own_keys, own_counts, flat, hc, hf, bk, bm, len(key), len(slot_keys), len(bk),
                      self.touched, dirty)

    def _dirty(self):
        nk, ok = neighbour_keys(self.touched)
        return nk[ok]

    def points(self):
        """(xyz, ids) in id order"""
        o = np.argsort(self.ids, kind="stable")
        return self.xyz[o], self.ids[o]

    def flagged_set(self):
        return set(map(tuple, self.flagged.tolist()))


# ---- a dump of the product's map ---------------------------------------------------------------------------------------
class Dump:
    """both tables ((slots, 8) and (block slots, 4) uint32), arena[0, arena_top) as (n, 4) uint32, the kMapCounters words, the
    touched and dirty lists of the last add (slot indices), and k"""

    def __init__(self, table, btable, arena, counters, touched, dirty, k):
        self.table, self.btable, self.arena = table, btable, arena.view(np.uint32).reshape(-1, 4)
        self.counters, self.touched, self.dirty, self.k = counters, touched, dirty, int(k)

    def live(self):
        return ~((self.table[:, 0] == EMPTY) & (self.table[:, 1] == EMPTY))

    def keys(self):
        return self.table[:, 0].astype(np.uint64) | (self.table[:, 1].astype(np.uint64) << np.uint64(32))

    def layout(self):
        if getattr(self, "_layout", None) is None:
            self._layout = self._make_layout()
        return self._layout

    def _make_layout(self):
        t, live = self.table, self.live()
        keys = self.keys()
        sl = np.nonzero(live)[0]
        sl = sl[np.argsort(keys[sl], kind="stable")]
        occ = sl[t[sl, 3] > 0]
        own_flat = self.arena[_gather_index(t[occ, 2], t[occ, 3])]
        halo_flat = self.arena[_gather_index(t[sl, 4], t[sl, 5])]
        bl = ~((self.btable[:, 0] == EMPTY) & (self.btable[:, 1] == EMPTY))
        bkeys = self.btable[bl, 0].astype(np.uint64) | (self.btable[bl, 1].astype(np.uint64) << np.uint64(32))
        bmask = self.btable[bl, 2].astype(np.uint64) | (self.btable[bl, 3].astype(np.uint64) << np.uint64(32))
        bo = np.argsort(bkeys)
        c = self.counters
        return Layout(keys[sl], keys[occ], t[occ, 3].astype(np.int64), own_flat, t[sl, 5].astype(np.int64), halo_flat,
                      bkeys[bo], bmask[bo], np.int32(np.uint32(c[CTR_POINTS])), c[CTR_SLOTS_USED], c[CTR_BLOCKS_USED],
                      np.unique(keys[self.touched]), np.unique(keys[self.dirty]))


def _chains_ok(table_keys, live, home):
    """every live key sits at or after its home slot with no empty slot between (linear probing, wrapping)"""
    n = len(live)
    empty2 = np.concatenate([~live, ~live]).astype(np.int64)
    cum = np.concatenate([[0], np.cumsum(empty2)])
    pos = np.nonzero(live)[0]
    h = home[pos].astype(np.int64)
    end = np.where(pos >= h, pos, pos + n)                    # the slot, unwrapped after the home
    return (cum[end + 1] - cum[h] == 0) & (end - h < 128)


def check_layout(d, halo=True):
    """the layout invariants of a Dump; returns a list of violations (empty: all hold).  halo=False leaves out the bucket
    check, for a caller that compares the buckets with a restatement built from the same own extents anyway"""
    bad = []
    t, live = d.table, d.live()
    keys = d.keys()
    slots = len(t)
    lk = keys[live]
    if len(np.unique(lk)) != len(lk):
        bad.append("duplicate voxel keys")
    if not _chains_ok(keys, live, voxel_hash(keys) & np.uint32(slots - 1)).all():
        bad.append("a voxel key is not reachable from its home slot")
    bl = ~((d.btable[:, 0] == EMPTY) & (d.btable[:, 1] == EMPTY))
    bkeys = d.btable[:, 0].astype(np.uint64) | (d.btable[:, 1].astype(np.uint64) << np.uint64(32))
    if len(np.unique(bkeys[bl])) != int(bl.sum()):
        bad.append("duplicate block keys")
    if not _chains_ok(bkeys, bl, block_home(bkeys) & np.uint32(len(d.btable) - 1)).all():
        bad.append("a block key is not reachable from its home slot")
    top = int(d.counters[CTR_ARENA_TOP])
    if len(d.arena) != top:
        bad.append("arena dump is not arena_top long")
    st, ct = np.concatenate([t[live, 2], t[live, 4]]).astype(np.int64), np.concatenate([t[live, 3], t[live, 5]]).astype(np.int64)
    used = ct > 0
    st, ct = st[used], ct[used]
    if (st < ARENA_FIRST).any() or (st + ct > top).any():
        bad.append("an extent lies outside [16, arena_top)")
    o = np.argsort(st, kind="stable")
    if ((st[o][1:] - (st[o] + ct[o])[:-1]) < 0).any():
        bad.append("two live extents overlap")
    caps = t[live, 6].astype(np.int64)
    if (t[live, 3] > (caps & 0xFFFF) * 4).any() or (t[live, 5] > (caps >> 16) * 8).any():
        bad.append("a count above its capacity")
    if (t[live, 7] != 0).any():
        bad.append("a flags word is not 0")
    lay = d.layout()
    xyz = lay.own_flat[:, :3].copy().view(np.float32)
    vb, _ = voxels(cells(xyz), d.k)
    if not np.array_equal(pack(vb), np.repeat(lay.own_keys, lay.own_counts)):
        bad.append("an own point does not key to its slot's voxel")
    if len(np.unique(lay.own_flat[:, 3])) != len(lay.own_flat):
        bad.append("duplicate point ids")
    if len(np.unique(d.dirty)) != len(d.dirty):
        bad.append("duplicate dirty slots")
    if len(np.unique(d.touched)) != len(d.touched):
        bad.append("duplicate touched slots")
    if halo:
        hc, hf = halo_of(lay.slot_keys, lay.own_keys, lay.own_counts, lay.own_flat)
        if not (np.array_equal(hc, lay.halo_counts) and np.array_equal(hf, lay.halo_flat)):
            bad.append("a halo bucket is not the concatenation of its neighbours' own extents")
    if len(lay.own_keys):
        need = dilate(lay.own_keys)
        if len(np.setdiff1d(need, lay.slot_keys)):
            bad.append("an occupied voxel misses a neighbour slot")
        bk, bm = blocks_of(lay.own_keys)
        if not (np.array_equal(bk, lay.block_keys) and np.array_equal(bm, lay.block_masks)):
            bad.append("block masks are not the occupancy of the voxels")
    if lay.points != len(lay.own_flat) or lay.slots_used != len(lay.slot_keys) or lay.blocks_used != len(lay.block_keys):
        bad.append("counters disagree with the tables")
    return bad
