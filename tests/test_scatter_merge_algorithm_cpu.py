"""The ALGORITHM of the hash-table gradient scatter's warp merge (ngp_pl_b200/csrc/network.cu: k_grid_scatter_merged),
replayed lane by lane on the CPU.

A warp holds 32 consecutive samples of one level. Lanes with equal cells form runs (an invalid lane is a run of its own);
each run is summed into its head. A valid head whose previous lane is valid and whose cell is adjacent to that lane's cell
(every |delta| <= 1) has a link: the corners the two cells share. Through the link of the NEXT head, a head hands to it
the corners they share, except the corners it shares with its own previous head; it issues the rest, x-pairs as one
16-byte reduction when both corners are issued and their entries are an aligned pair, as 8-byte reductions otherwise.
The receiver adds what it was handed into its own corners and issues them.

This file restates that control flow (the kernel's bit masks, corner shifts and shared-memory slots) and holds the
entries it issues to a plain per-sample, per-corner float64 sum: every contribution counted once, per-entry sums equal.
Synthetic warps cover each kind of adjacency (face, edge, vertex), jumps of 2 cells, runs of one cell, runs that span
two rays, invalid lanes, the dense levels' wrap at the upper boundary and hashed levels where distinct vertices collide.
Test infrastructure only.
"""
import numpy as np
import pytest

P1, P2 = 2654435761, 805459861
M32 = 0xFFFFFFFF


def _vertex_entry(vx, vy, vz, res, entries, hashed):
    """the table entry of one grid vertex, as grid_corner_index (uint32 arithmetic)"""
    vx, vy, vz = vx & M32, vy & M32, vz & M32
    if hashed:
        return (vx ^ ((vy * P1) & M32) ^ ((vz * P2) & M32)) & (entries - 1)
    i = (vx + vy * res + vz * res * res) & M32
    i = i - entries if i >= entries else i
    return min(i, entries - 1)


def _cell_entries(c, res, entries, hashed):
    """the 8 corner entries of a cell, k = dx + 2 dy + 4 dz, as grid_corner_indices (per-axis terms shared)"""
    gx, gy, gz = (int(t) & M32 for t in c)
    out = []
    if hashed:
        mask = entries - 1
        y0 = (gy * P1) & M32
        z0 = (gz * P2) & M32
        ys, zs = (y0, (y0 + P1) & M32), (z0, (z0 + P2) & M32)
        for k in range(8):
            out.append(((gx + (k & 1)) & M32 ^ ys[(k >> 1) & 1] ^ zs[k >> 2]) & mask)
    else:
        r2 = (res * res) & M32
        b00 = (gx + gy * res + gz * r2) & M32
        for k in range(8):
            v = (b00 + (k & 1) + ((k >> 1) & 1) * res + (k >> 2) * r2) & M32
            v = v - entries if v >= entries else v
            out.append(min(v, entries - 1))
    return out


def _shared(d):
    """grid_shared_corners: corners k of a cell that are corners of the cell + d"""
    m = 0xFF
    for ax, (lo, hi) in enumerate(((0x55, 0xAA), (0x33, 0xCC), (0x0F, 0xF0))):
        m &= hi if d[ax] > 0 else lo if d[ax] < 0 else 0xFF
    return m


def _delta(a, b):
    """b - a per axis as the kernel's (int)(uint32 - uint32)"""
    out = []
    for i in range(3):
        v = (int(b[i]) - int(a[i])) & M32
        out.append(v - (1 << 32) if v >= 1 << 31 else v)
    return out


def warp_merge(cells, valid, contrib, res, entries, hashed):
    """one warp at one level. cells: 32 cells (x, y, z); valid: 32 bools; contrib: (32, 8, 2) float64 corner contributions.
    -> (issued: list of (entry, value float64 (2,), reduction kind "v4" / "v2")), the kernel's reductions in any order"""
    valid = [bool(v) for v in valid]
    cells = [tuple(int(t) & M32 for t in c) for c in cells]
    head = [l == 0 or not valid[l] or not valid[l - 1] or cells[l] != cells[l - 1] for l in range(32)]
    run_end = [0] * 32
    for l in range(32):
        e = l
        while e + 1 < 32 and not head[e + 1]:
            e += 1
        run_end[l] = e
    acc = np.array(contrib, dtype=np.float64).copy()
    for l in range(32):  # the segmented reduction: each head holds its run's sum
        if head[l]:
            acc[l] = acc[l:run_end[l] + 1].sum(axis=0)
    link = [0] * 32
    for l in range(32):
        if valid[l] and l > 0 and valid[l - 1] and head[l]:
            o = _delta(cells[l], cells[l - 1])
            if all(abs(t) <= 1 for t in o):
                link[l] = _shared(o) | (o[0] + 2 * o[1] + 4 * o[2] + 8) << 8
    s_hand = np.full((32, 9, 2), np.nan)
    fwd, fwd_out = [0] * 32, [0] * 32
    for l in range(32):
        nlink = link[(run_end[l] + 1) & 31]
        if valid[l] and head[l] and nlink:
            o = (nlink >> 8) - 8
            mine = link[l] & 0xFF
            fwd_out[l] = nlink & 0xFF & ~((mine << o) if o >= 0 else (mine >> -o)) & M32
            fwd[l] = fwd_out[l] >> o if o >= 0 else (fwd_out[l] << -o) & M32
            for k in range(8):
                if (fwd[l] >> k) & 1:
                    assert 0 <= k + o < 8
                    s_hand[run_end[l] + 1, k + o] = acc[l, k]
    issued = []
    for l in range(32):
        if not (valid[l] and head[l]):
            continue
        ph = 0 if l == 0 else max(j for j in range(l) if head[j])
        recv = fwd_out[ph]
        for k in range(8):
            if link[l] and (recv >> k) & 1:
                assert not np.isnan(s_hand[l, k]).any()
                acc[l, k] += s_hand[l, k]
        own = 0xFF & ~fwd[l]
        idx = _cell_entries(cells[l], res, entries, hashed)
        for k in range(0, 8, 2):
            o0, o1 = (own >> k) & 1, (own >> (k + 1)) & 1
            if o0 and o1 and (idx[k] ^ idx[k + 1]) == 1:
                issued.append((idx[k], acc[l, k], "v4"))
                issued.append((idx[k + 1], acc[l, k + 1], "v4"))
            else:
                if o0:
                    issued.append((idx[k], acc[l, k], "v2"))
                if o1:
                    issued.append((idx[k + 1], acc[l, k + 1], "v2"))
    return issued


def _reference(cells, valid, contrib, res, entries, hashed):
    ref = {}
    for l in range(32):
        if not valid[l]:
            continue
        for k in range(8):
            e = _vertex_entry(int(cells[l][0]) + (k & 1), int(cells[l][1]) + ((k >> 1) & 1), int(cells[l][2]) + (k >> 2),
                              res, entries, hashed)
            ref[e] = ref.get(e, 0.0) + contrib[l, k]
    return ref


def _run_and_check(cells, valid, res, entries, hashed, rng):
    cells = np.asarray(cells, dtype=np.int64)
    valid = np.asarray(valid, dtype=bool)
    # integer contributions: every sum is exact, so "counted once" is an equality
    contrib = rng.randint(-1000, 1001, (32, 8, 2)).astype(np.float64)
    issued = warp_merge(cells, valid, contrib, res, entries, hashed)
    got = {}
    for e, v, _ in issued:
        got[e] = got.get(e, 0.0) + v
    ref = _reference(cells, valid, contrib, res, entries, hashed)
    assert set(got) == set(ref)
    for e in ref:
        assert np.array_equal(got[e], ref[e]), (e, got[e], ref[e])
    # float contributions against float64 in the kernel's float32 partial sums' reach
    contrib = rng.standard_normal((32, 8, 2))
    issued = warp_merge(cells, valid, contrib, res, entries, hashed)
    ref = _reference(cells, valid, contrib, res, entries, hashed)
    got = {}
    for e, v, _ in issued:
        got[e] = got.get(e, 0.0) + v
    for e in ref:
        np.testing.assert_allclose(got[e], ref[e], rtol=0, atol=1e-12)
    return issued


def _issue_count(issued):
    return sum(1 for *_, kind in issued if kind == "v2") + sum(1 for *_, kind in issued if kind == "v4") // 2


HASHED = dict(res=1025, entries=1 << 19, hashed=True)
DENSE = dict(res=65, entries=65 ** 3 + 7 & ~7, hashed=False)


def _walk(start, steps):
    cells = [tuple(start)]
    for s in steps:
        cells.append(tuple(a + b for a, b in zip(cells[-1], s)))
    return cells


@pytest.mark.parametrize("level", ["hashed", "dense"])
@pytest.mark.parametrize("kind,step,saved", [
    ("face", (1, 0, 0), 4), ("face_y", (0, -1, 0), 4), ("edge", (1, 1, 0), 2), ("edge_xz", (-1, 0, 1), 2),
    ("vertex", (1, -1, 1), 1), ("jump2", (2, 0, 0), 0), ("jump2_diag", (1, 2, 0), 0)])
def test_adjacency_kinds(level, kind, step, saved):
    """two runs of 16 lanes: the second run's cell is the first's + step; `saved` corners are handed over"""
    rng = np.random.RandomState(sum(map(ord, kind + level)))
    p = HASHED if level == "hashed" else DENSE
    a = (20, 30, 40)
    b = tuple(x + s for x, s in zip(a, step))
    cells = [a] * 16 + [b] * 16
    issued = _run_and_check(cells, [True] * 32, p["res"], p["entries"], p["hashed"], rng)
    assert len(issued) == 16 - saved  # corner contributions that reach memory


def test_same_cell_is_one_run():
    rng = np.random.RandomState(1)
    issued = _run_and_check([(7, 8, 9)] * 32, [True] * 32, **HASHED, rng=rng)
    assert len(issued) == 8


def test_chain_receives_and_forwards_in_one_pass():
    """a walk of single-lane runs: heads that receive from the previous head and hand on to the next; a corner shared
    with both neighbours is issued by the middle head"""
    rng = np.random.RandomState(2)
    steps = [(1, 0, 0), (0, 1, 0), (1, 1, 0), (0, 0, 1), (-1, 0, 0), (1, 1, 1), (0, -1, 0)] * 5
    cells = _walk((100, 200, 300), steps[:31])
    for p in (HASHED, DENSE):
        issued = _run_and_check([(c[0] % 60, c[1] % 60, c[2] % 60) for c in cells] if not p["hashed"] else cells,
                                [True] * 32, p["res"], p["entries"], p["hashed"], rng)
        assert len(issued) < 8 * 32


def test_runs_spanning_two_rays():
    """the last samples of one ray and the first of the next: an arbitrary jump, or by chance an adjacent cell"""
    rng = np.random.RandomState(3)
    ray_a = _walk((10, 10, 10), [(1, 0, 0), (0, 0, 0), (0, 1, 0), (0, 0, 0), (1, 0, 0)] * 3)[:16]
    for ray_b_start in ((500, 3, 77), (ray_a[-1][0] + 1, ray_a[-1][1], ray_a[-1][2] - 1), ray_a[-1]):
        ray_b = _walk(ray_b_start, [(0, 0, 0), (0, 0, 1), (0, 0, 0), (1, 1, 0)] * 4)[:16]
        _run_and_check(ray_a + ray_b, [True] * 32, **HASHED, rng=rng)


@pytest.mark.parametrize("pattern", ["middle", "tail", "alternate", "lane0", "all"])
def test_invalid_lanes(pattern):
    rng = np.random.RandomState(sum(map(ord, pattern)))
    cells = _walk((5, 6, 7), [(1, 0, 0), (0, 0, 0), (0, 1, 0), (1, 0, 1), (0, 0, 0), (0, 0, 0)] * 6)[:32]
    valid = np.ones(32, bool)
    if pattern == "middle":
        valid[[9, 10, 20]] = False
    elif pattern == "tail":
        valid[23:] = False
    elif pattern == "alternate":
        valid[1::2] = False
    elif pattern == "lane0":
        valid[0] = False
    else:
        valid[:] = False
    issued = _run_and_check(cells, valid, **HASHED, rng=rng)
    if pattern == "all":
        assert issued == []


def test_dense_wrap_at_the_upper_boundary():
    """cells at res - 1 on a dense level: their +1 corners wrap past the level's end (and are clamped); the neighbour that
    shares them must reach the same entries"""
    rng = np.random.RandomState(4)
    res = 17
    entries = (res ** 3 + 7) // 8 * 8
    cells = _walk((res - 2, res - 1, res - 1), [(1, 0, 0), (0, 0, 0), (0, -1, 0), (-1, 0, 0), (0, 0, 0), (1, 0, -1),
                                                 (0, 0, 1), (0, 1, 0)] * 4)[:32]
    _run_and_check(cells, [True] * 32, res, entries, False, rng)
    # outside the unit cube too: cells past the level, where the clamp, not the wrap, decides the entry
    cells = _walk((res, res, res - 1), [(1, 0, 0), (0, 1, 0), (0, 0, 1), (-1, -1, 0)] * 8)[:32]
    _run_and_check(cells, [True] * 32, res, entries, False, rng)


def test_hash_collision_of_distinct_vertices():
    """a tiny hashed table where distinct vertices share an entry: only equal vertices are merged, the colliding ones
    still land in their common entry"""
    rng = np.random.RandomState(5)
    entries = 1 << 5
    cells = _walk((3, 4, 5), [(1, 0, 0), (0, 1, 0), (0, 0, 1), (1, 1, 1), (-1, 0, 0), (0, 0, 0)] * 6)[:32]
    ent = [_vertex_entry(c[0] + (k & 1), c[1] + ((k >> 1) & 1), c[2] + (k >> 2), 1025, entries, True)
           for c in cells for k in range(8)]
    verts = {(c[0] + (k & 1), c[1] + ((k >> 1) & 1), c[2] + (k >> 2)) for c in cells for k in range(8)}
    assert len(set(ent)) < len(verts)  # collisions happen
    _run_and_check(cells, [True] * 32, 1025, entries, True, rng)


@pytest.mark.parametrize("seed", range(12))
def test_random_walks(seed):
    """random walks of cells with runs, jumps and invalid lanes, on hashed (small tables: collisions) and dense levels"""
    rng = np.random.RandomState(100 + seed)
    for p in (dict(res=1025, entries=1 << 7, hashed=True), HASHED, dict(res=9, entries=736, hashed=False), DENSE):
        steps = rng.randint(-1, 2, (31, 3))
        steps[rng.rand(31) < 0.3] = 0
        jump = rng.rand(31) < 0.1
        steps[jump] = rng.randint(-3, 4, (int(jump.sum()), 3))
        start = rng.randint(0, p["res"], 3)
        cells = _walk(tuple(start), [tuple(s) for s in steps])
        valid = rng.rand(32) > 0.1
        _run_and_check(cells, valid, p["res"], p["entries"], p["hashed"], rng)


def test_face_crossings_issue_fewer_reductions():
    """runs of 2 lanes stepping one face at a time along y: each head hands 4 corners (2 aligned x-pairs) on"""
    rng = np.random.RandomState(6)
    cells = [c for c in _walk((40, 40, 40), [(0, 1, 0)] * 15) for _ in range(2)]
    issued = _run_and_check(cells, [True] * 32, **HASHED, rng=rng)
    # 16 cells; 15 hand-overs of 2 pairs each; gx = 40 is even, so every issued pair is one 16-byte reduction
    assert _issue_count(issued) == 16 * 4 - 15 * 2
