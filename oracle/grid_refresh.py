"""numpy restatement of the occupancy-grid refresh -- TEST INFRASTRUCTURE ONLY (no torch, no GPU).

ngp_update_density_grid = ngp_update_density_grid_pick + ngp_update_density_grid_eval in ngp_pl_b200/csrc/train.cu,
the device version of the reference's NGP.update_density_grid + sample_uniform_and_occupied_cells (networks.py:169-195,
240-269). One function per stage; what is exact and what is bounded:

  pcg_hash, u01, refresh_seed     exact (uint32)                   train.cu pcg_hash / u01, Trainer._refresh_seed
  pick_keys                       exact                            k_grid_flags + cub Flagged + k_grid_pick_cells
  cascade_cells                   exact (np.unique = radix sort + cub Unique), tot[c] the running slot base
  jitter                          bit for bit                      k_grid_jitter
  jitter_reference                float64 formula of networks.py:250-253 + 2 ulp(s) bound
  merge                           bit for bit without erode; float64 + bound with erode       k_grid_merge
  mean                            float64 + bound of the kernel's fp32 sum chain              k_grid_merge + k_grid_mean
  threshold, packbits             exact                            k_packbits_f32x4 with thr_dev = &stats[2]

Jitter arithmetic, read from `cuobjdump -sass` of k_grid_jitter built with the project's flags (-O3, sm_90a, no
fast-math): per axis one MUFU.RCP + FFMA Newton sequence with the FCHK / slow-path call of IEEE division for cc / (G-1),
FFMA q*2 - 1 (exact: q*2 is exact), FADD s - half, FMUL for the centre, FFMA u01*2 - 1 (exact), and one FFMA
(u01*2 - 1) * half + centre -- the final multiply-add is contracted, the centre product is not. So
    centre = fl(fl(fl(cc / (G-1)) * 2 - 1) * fl(s - half)),   x = fma(u01 * 2 - 1, half, centre)
with s = fminf(2^(c-1), scale) and half = fl(s / G) in fp32. The fma is restated with the exact float64 product and a
TwoSum residual, as oracle/grad64.py: ray_positions does.

Erode bound (k_grid_merge with count_grid): d = fminf(fmaxf(powf(decay, 1.0f / count), 0.1f), 0.95f). The CUDA C++
Programming Guide (12.9), appendix "Mathematical Functions", table "Single-Precision Mathematical Standard Library
Functions with Maximum ULP Error", gives powf(x, y) a maximum error of 4 ulp (full range). 1.0f / count is an IEEE
division, rounded once: it moves decay^y by at most |ln decay| * y * 2^-24 relative. The clamp is 1-Lipschitz, the
product g * d is rounded once more (2^-24 relative), and max(., tmp) is 1-Lipschitz.

Mean bound: sum of the positive cells in fp32 along a chain of depth k = ceil(n / (blocks * 256)) per-thread serial
terms + 5 warp shuffles + 8 warps + ceil(blocks / 256) per-thread partials in k_grid_mean + 8 tree levels, + 1 for
the division: |mean32 - mean64| <= gamma_k * sum / count (gamma_k = k u / (1 - k u), u = 2^-24), plus 2^-24 of the
mean once count > 2^24 (the (float)count conversion). No positive cell: NaN, as the reference's empty .mean().
"""
import numpy as np

U = 2.0 ** -24           # unit roundoff of float32
POWF_ULP = 4             # powf maximum error, CUDA C++ Programming Guide (see above)
MERGE_MAX_BLOCKS = 2048  # train.cu


# ---------------------------------------------------------------------------------------------------
# integer hashing
# ---------------------------------------------------------------------------------------------------
def pcg_hash(v):
    """train.cu pcg_hash, uint32 in, uint32 out (array or scalar)"""
    v = np.asarray(v, dtype=np.uint32)
    with np.errstate(over="ignore"):
        s = v * np.uint32(747796405) + np.uint32(2891336453)
        w = ((s >> ((s >> np.uint32(28)) + np.uint32(4))) ^ s) * np.uint32(277803737)
    return (w >> np.uint32(22)) ^ w


def u01(h):
    """train.cu u01: (h >> 8) * 2^-24 in float32 (exact)"""
    return (np.asarray(h, dtype=np.uint32) >> np.uint32(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)


def refresh_seed(seed, step):
    """Trainer._refresh_seed"""
    return (int(seed) * 2654435761 + int(step) * 40503 + 12345) & 0xffffffff


def slot_hash(seed, c, i):
    """h of slot / rank i of cascade c: pcg_hash(seed ^ pcg_hash(i + 0x9e3779b9 (c + 1))) (k_grid_pick_cells, k_grid_jitter)"""
    i = np.asarray(i, dtype=np.uint32)
    with np.errstate(over="ignore"):
        a = i + np.uint32((0x9e3779b9 * (c + 1)) & 0xffffffff)
    return pcg_hash(np.uint32(seed) ^ pcg_hash(a))


# ---------------------------------------------------------------------------------------------------
# Morton order (march.cuh morton_spread10 / morton_compact10)
# ---------------------------------------------------------------------------------------------------
def _spread10(v):
    v = np.asarray(v, dtype=np.uint32) & np.uint32(0x3ff)
    v = (v | (v << np.uint32(16))) & np.uint32(0x030000ff)
    v = (v | (v << np.uint32(8))) & np.uint32(0x0300f00f)
    v = (v | (v << np.uint32(4))) & np.uint32(0x030c30c3)
    return (v | (v << np.uint32(2))) & np.uint32(0x09249249)


def _compact10(v):
    v = np.asarray(v, dtype=np.uint32) & np.uint32(0x09249249)
    v = (v | (v >> np.uint32(2))) & np.uint32(0x030c30c3)
    v = (v | (v >> np.uint32(4))) & np.uint32(0x0300f00f)
    v = (v | (v >> np.uint32(8))) & np.uint32(0x030000ff)
    return (v | (v >> np.uint32(16))) & np.uint32(0x3ff)


def morton_encode(x, y, z):
    return _spread10(x) | (_spread10(y) << np.uint32(1)) | (_spread10(z) << np.uint32(2))


def morton_decode(m):
    """(n, 3) uint32 coordinates of Morton indices m: x from bits 0, 3, 6..., y from 1, 4..., z from 2, 5..."""
    m = np.asarray(m, dtype=np.uint32)
    return np.stack([_compact10(m), _compact10(m >> np.uint32(1)), _compact10(m >> np.uint32(2))], -1)


# ---------------------------------------------------------------------------------------------------
# picks
# ---------------------------------------------------------------------------------------------------
def uniform_coords(seed, c, G, M):
    """(M, 3) coordinates of the uniform picks, slots [0, M) (k_grid_pick_cells, networks.py:182-184)"""
    h = slot_hash(seed, c, np.arange(M, dtype=np.uint32))
    G = np.uint32(G)
    return np.stack([pcg_hash(h) % G, pcg_hash(h ^ np.uint32(0x68bc21eb)) % G,
                     pcg_hash(h ^ np.uint32(0x02e5be93)) % G], -1)


def occupied_list(grid_c, thr):
    """k_grid_flags (grid > thr, strict, in float32) + cub DeviceSelect::Flagged (stable: index order)"""
    return np.flatnonzero(np.asarray(grid_c, np.float32) > np.float32(thr)).astype(np.uint32)


def pick_keys(grid_c, thr, seed, c, G):
    """the 2M keys of cascade c in slot order: [0, M) uniform cells, [M, 2M) occupied cells (G^3 when there is none)
    (k_grid_pick_cells, networks.py:185-192); also returns the occupied list and the occupied draws' list indices"""
    g3 = G ** 3
    M = g3 // 4
    xyz = uniform_coords(seed, c, G, M)
    uni = morton_encode(xyz[:, 0], xyz[:, 1], xyz[:, 2])
    occ = occupied_list(grid_c, thr)
    h = slot_hash(seed, c, np.arange(M, 2 * M, dtype=np.uint32))
    if occ.size == 0:
        draw = None
        occ_keys = np.full(M, g3, dtype=np.uint32)
    else:
        draw = pcg_hash(h ^ np.uint32(0x7feb352d)) % np.uint32(occ.size)
        occ_keys = occ[draw]
    return np.concatenate([uni, occ_keys]).astype(np.uint32), occ, draw


def cascade_cells(grid, thr, seed, G, warmup):
    """per cascade the cells the refresh evaluates, in slot order: warm-up every cell (slot i = cell i), else the
    cascade's picks sorted and de-duplicated (cub radix sort + Unique == np.unique). Returns (cells, tot): cells[c] uint32
    (G^3 = the "none" key), tot[c] = first slot of cascade c, tot[C] = number of slots."""
    C = grid.shape[0]
    g3 = G ** 3
    cells, tot = [], [0]
    for c in range(C):
        k = np.arange(g3, dtype=np.uint32) if warmup else np.unique(pick_keys(grid[c], thr, seed, c, G)[0])
        cells.append(k)
        tot.append(tot[-1] + k.size)
    return cells, np.array(tot, dtype=np.int64)


def cell_index(cells, G):
    """cell_idx of every slot: c G^3 + cell, -1 for the "none" key"""
    g3 = G ** 3
    out = [np.where(k >= g3, -1, c * g3 + k.astype(np.int64)) for c, k in enumerate(cells)]
    return np.concatenate(out).astype(np.int32)


# ---------------------------------------------------------------------------------------------------
# jitter
# ---------------------------------------------------------------------------------------------------
def cascade_extent(c, scale, G):
    """s = fminf(scalbnf(1, c - 1), scale), half = s / G, both float32"""
    s = np.minimum(np.float32(2.0 ** (c - 1)), np.float32(scale))
    return s, np.float32(s / np.float32(G))


def fma32(a, b, c):
    """fmaf(a, b, c) of float32 arrays, bit for bit: the float64 product is exact; the float64 sum is rounded at most
    once and TwoSum gives its residual; rounding it to float32 is the fma's result unless it lies exactly halfway
    between two floats while the residual is not 0 -- then the fma rounds towards the residual."""
    a, b, c = (np.asarray(v, np.float32) for v in (a, b, c))
    p = a.astype(np.float64) * b.astype(np.float64)
    o = np.broadcast_to(c.astype(np.float64), p.shape)
    s = p + o
    bp = s - o
    res = (p - bp) + (o - (s - bp))
    x = s.astype(np.float32)
    xd = x.astype(np.float64)
    nb = np.where(s > xd, np.nextafter(x, np.float32(np.inf)), np.nextafter(x, np.float32(-np.inf)))
    tie = (s != xd) & ((s - xd) == (nb.astype(np.float64) - s)) & (res != 0)
    x = np.where(tie & (res > 0), np.maximum(x, nb), np.where(tie & (res < 0), np.minimum(x, nb), x))
    return x.astype(np.float32)


def jitter_offsets(seed, c, n):
    """u01 of the three axes' hashes of ranks [0, n): h = pcg_hash(h + 0x85ebca6b) per axis, (n, 3) float32"""
    h = slot_hash(seed, c, np.arange(n, dtype=np.uint32))
    out = []
    for _ in range(3):
        with np.errstate(over="ignore"):
            h = pcg_hash(h + np.uint32(0x85ebca6b))
        out.append(u01(h))
    return np.stack(out, -1)


def jitter(cells_c, seed, c, G, scale):
    """k_grid_jitter for one cascade, bit for bit: (n, 3) float32 points, 0 for the "none" key"""
    g3 = G ** 3
    n = cells_c.size
    cc = morton_decode(np.minimum(cells_c, g3 - 1)).astype(np.float32)
    s, half = cascade_extent(c, scale, G)
    q = (cc.astype(np.float64) / np.float64(np.float32(G - 1))).astype(np.float32)  # IEEE division (exact in float64)
    a = (q * np.float32(2.0) - np.float32(1.0)).astype(np.float32)
    centre = (a * np.float32(s - half)).astype(np.float32)
    o = (jitter_offsets(seed, c, n) * np.float32(2.0) - np.float32(1.0)).astype(np.float32)
    x = fma32(o, half, centre)
    x[cells_c >= g3] = 0
    return x


def refresh_points(cells, seed, G, scale):
    return np.concatenate([jitter(k, seed, c, G, scale) for c, k in enumerate(cells)]).reshape(-1, 3)


def jitter_reference(cells_c, seed, c, G, scale):
    """networks.py:250-253 in float64 with the same u: (coords / (G-1) * 2 - 1) * (s - half) + (u * 2 - 1) * half, and
    the bound 2 ulp(s) = 2^-22 s on the float32 point (|a - a64| <= 2^-24 from the rounded quotient, the centre product
    and the fma round once each, |centre|, |x| <= s), plus how far float32 moved s - half and half (0 when exact)"""
    cc = morton_decode(cells_c).astype(np.float64)
    s = min(2.0 ** (c - 1), float(scale))
    half = s / G
    u = jitter_offsets(seed, c, cells_c.size).astype(np.float64)
    x = (cc / (G - 1) * 2 - 1) * (s - half) + (u * 2 - 1) * half
    s32, h32 = cascade_extent(c, scale, G)
    extra = abs(float(np.float32(s32 - h32)) - (s - half)) + abs(float(h32) - half) + abs(float(s32) - s)
    return x, 2.0 ** -22 * s + 2 * extra


def cell_box(cells_c, c, G, scale):
    """cell k's box [-s + k 2s/G, -s + (k+1) 2s/G] per axis, float64, (n, 3) each"""
    cc = morton_decode(cells_c).astype(np.float64)
    s = min(2.0 ** (c - 1), float(scale))
    return -s + cc * 2 * s / G, -s + (cc + 1) * 2 * s / G


# ---------------------------------------------------------------------------------------------------
# merge, mean, threshold, bits
# ---------------------------------------------------------------------------------------------------
def scatter(cell_idx, sigma, shape):
    """k_grid_scatter: tmp = 0 except tmp[cell_idx] = sigma (each cell appears at most once)"""
    tmp = np.zeros(int(np.prod(shape)), np.float32)
    live = cell_idx >= 0
    tmp[cell_idx[live]] = sigma[live]
    return tmp.reshape(shape)


def merge(grid, tmp, decay):
    """k_grid_merge without erode, bit for bit: g < 0 ? g : max(fl(g decay), tmp)"""
    g = np.asarray(grid, np.float32)
    return np.where(g < 0, g, np.maximum((g * np.float32(decay)).astype(np.float32), tmp)).astype(np.float32)


def erode_decay(count, decay):
    """float64 clamp(decay^(1/count), 0.1, 0.95) and the bound on the kernel's float32 d (see the module docstring);
    count = 0 gives d = 0.1 exactly (bound 0)"""
    count = np.asarray(count, np.float32).astype(np.float64)
    dec = float(np.float32(decay))
    with np.errstate(divide="ignore", over="ignore"):
        y = 1.0 / count
        p = np.power(dec, y)
    d = np.clip(p, float(np.float32(0.1)), float(np.float32(0.95)))
    with np.errstate(invalid="ignore"):
        bd = p * (abs(np.log(dec)) * y * U + POWF_ULP * 2.0 ** -23)
    bd = np.where(np.isfinite(bd), bd, 0.0)
    # a clamped powf within its own bound of the clamp lands on the clamp: the bound carries over unchanged
    return d, bd


def merge_erode(grid, tmp, count, decay):
    """k_grid_merge with count_grid: float64 value and bound per cell (-1 cells stay -1 exactly, bound 0)"""
    g = np.asarray(grid, np.float32).astype(np.float64)
    d, bd = erode_decay(count, decay)
    gd = g * d
    val = np.where(g < 0, g, np.maximum(gd, np.asarray(tmp, np.float64)))
    bound = np.where(g < 0, 0.0, np.abs(g) * bd + U * np.abs(gd) * (1 + bd))
    return val, bound


def gamma(k):
    return k * U / (1 - k * U)


def mean_depth(n_cells, n_blocks):
    """depth of k_grid_merge + k_grid_mean's fp32 sum chain, + 1 for the division"""
    return -(-n_cells // (n_blocks * 256)) + 5 + 8 + -(-n_blocks // 256) + 8 + 1


def merge_blocks(n_cells, sm_count):
    """k_grid_merge's grid size: ceil(n / 256) capped at 8 blocks per SM and MERGE_MAX_BLOCKS"""
    return min(-(-n_cells // 256), sm_count * 8, MERGE_MAX_BLOCKS)


def mean(grid, n_blocks):
    """float64 mean of the positive cells (NaN if none) and the bound on the kernel's float32 mean"""
    g = np.asarray(grid, np.float32).reshape(-1)
    pos = g[g > 0].astype(np.float64)
    if pos.size == 0:
        return float("nan"), 0.0
    tot = float(pos.sum())
    m = tot / pos.size
    bound = gamma(mean_depth(g.size, n_blocks)) * m
    if pos.size > 2 ** 24:
        bound += U * m
    return m, bound


def threshold(thr, mean32):
    """k_packbits's fminf(thr, *thr_dev) in float32: a NaN mean gives thr"""
    thr = np.float32(thr)
    m = np.float32(mean32)
    return thr if np.isnan(m) else np.minimum(thr, m)


def packbits(grid, thr):
    """bit i % 8 of byte i / 8 = grid[i] > thr (float32 compare)"""
    g = np.asarray(grid, np.float32).reshape(-1)
    return np.packbits(g > np.float32(thr), bitorder="little")
