// Occupancy-grid ray marcher core: the device functions shared by every kernel that marches, and the host-side
// choice of which specialisation to launch.
//
// Parity contract: the per-ray sequence of (t, dt, xyz) must be BIT-EXACT with the reference's
// raymarching_train_kernel / raymarching_test_kernel (reference models/csrc/raymarching.cu:166-280,
// :335-404). The reference is compiled with nvcc's default -fmad=true and no fast-math; which
// multiplies/adds get fused there is read off its SASS (SURVEY.md Appendix C). Here every rounding
// step is spelled with an explicit intrinsic (__fmaf_rn / __fmul_rn / __fadd_rn / __fdiv_rn), so the
// result does not depend on how the compiler chooses to contract the surrounding code.
#pragma once
#include <type_traits>
#include "common.cuh"

struct MarchConst {
    const uint8_t* __restrict__ bitfield;  // cascades * G^3 / 8 bytes, bit i%8 of byte i/8, i = mip*G^3 + morton(x,y,z)
    int cascades;
    int grid_size;
    int max_samples;
    uint32_t grid_size3;
    float scale;         // scene half extent (reference NGP.scale)
    float esf;           // exp_step_factor
    float dt_lo, dt_hi;  // clamp bounds of the step (reference raymarching.cu:11-13)
    float gs_f, gs_inv, gs_m1;
    float mb0, mb0_inv;  // mip 0: min(2^-1, scale) and its reciprocal (all a single-cascade grid ever uses)
};

// dt_scale is what the reference hands to calc_dt as `scale`: NGP.scale for the train kernel
// (raymarching.cu:196,207,231) but `cascades` for the test kernel (raymarching.cu:370,399).
__device__ __forceinline__ MarchConst make_march_const(const uint8_t* bitfield, int cascades, int grid_size,
                                                       int max_samples, float scale, float esf, float dt_scale) {
    MarchConst c;
    c.bitfield = bitfield;
    c.cascades = cascades;
    c.grid_size = grid_size;
    c.max_samples = max_samples;
    c.grid_size3 = (uint32_t)grid_size * (uint32_t)grid_size * (uint32_t)grid_size;
    c.scale = scale;
    c.esf = esf;
    c.gs_f = (float)grid_size;
    c.gs_inv = __fdiv_rn(1.0f, c.gs_f);
    c.gs_m1 = __fadd_rn(c.gs_f, -1.0f);
    c.dt_lo = __fdiv_rn(1.73205080757f, (float)max_samples);
    c.dt_hi = __fdiv_rn(__fmul_rn(dt_scale, 3.46410161514f), c.gs_f);
    c.mb0 = fminf(0.5f, scale);
    c.mb0_inv = __fdiv_rn(1.0f, c.mb0);
    return c;
}

__device__ __forceinline__ float march_dt(float t, const MarchConst& c) {
    // clamp(t*esf, lo, hi) == fmaxf(lo, fminf(t*esf, hi))
    return fmaxf(c.dt_lo, fminf(__fmul_rn(t, c.esf), c.dt_hi));
}

// spread the low 10 bits of v so that there are two zero bits between consecutive bits
__device__ __host__ __forceinline__ uint32_t morton_spread10(uint32_t v) {
    v &= 0x000003ffu;
    v = (v | (v << 16)) & 0x030000ffu;
    v = (v | (v << 8)) & 0x0300f00fu;
    v = (v | (v << 4)) & 0x030c30c3u;
    v = (v | (v << 2)) & 0x09249249u;
    return v;
}
__device__ __host__ __forceinline__ uint32_t morton_encode3(uint32_t x, uint32_t y, uint32_t z) {
    return morton_spread10(x) | (morton_spread10(y) << 1) | (morton_spread10(z) << 2);
}
__device__ __host__ __forceinline__ uint32_t morton_compact10(uint32_t v) {
    v &= 0x09249249u;
    v = (v | (v >> 2)) & 0x030c30c3u;
    v = (v | (v >> 4)) & 0x0300f00fu;
    v = (v | (v >> 8)) & 0x030000ffu;
    v = (v | (v >> 16)) & 0x000003ffu;
    return v;
}

struct MarchRay {
    float ox, oy, oz;
    float dx, dy, dz;
    float ix, iy, iz;  // IEEE 1/d
    float sx, sy, sz;  // copysign(1, d)
};

__device__ __forceinline__ MarchRay make_march_ray(float ox, float oy, float oz, float dx, float dy, float dz) {
    MarchRay r;
    r.ox = ox; r.oy = oy; r.oz = oz;
    r.dx = dx; r.dy = dy; r.dz = dz;
    r.ix = __fdiv_rn(1.0f, dx); r.iy = __fdiv_rn(1.0f, dy); r.iz = __fdiv_rn(1.0f, dz);
    r.sx = copysignf(1.0f, dx); r.sy = copysignf(1.0f, dy); r.sz = copysignf(1.0f, dz);
    return r;
}

// Slab test against one axis-aligned box (reference intersection.cu:5-22, :45-52), followed by the
// near-plane clamp render() applies (reference rendering.py:29). Returns (t1,t2), (-1,-1) on a miss.
__device__ __forceinline__ float2 ray_aabb(const MarchRay& r, float cx, float cy, float cz, float hx, float hy, float hz) {
    const float ax = __fmul_rn(__fsub_rn(__fsub_rn(cx, hx), r.ox), r.ix);
    const float bx = __fmul_rn(__fsub_rn(__fadd_rn(cx, hx), r.ox), r.ix);
    const float ay = __fmul_rn(__fsub_rn(__fsub_rn(cy, hy), r.oy), r.iy);
    const float by = __fmul_rn(__fsub_rn(__fadd_rn(cy, hy), r.oy), r.iy);
    const float az = __fmul_rn(__fsub_rn(__fsub_rn(cz, hz), r.oz), r.iz);
    const float bz = __fmul_rn(__fsub_rn(__fadd_rn(cz, hz), r.oz), r.iz);
    const float t1 = fmaxf(fmaxf(fminf(ax, bx), fminf(ay, by)), fminf(az, bz));
    const float t2 = fminf(fminf(fmaxf(ax, bx), fmaxf(ay, by)), fmaxf(az, bz));
    if (t1 > t2) return make_float2(-1.0f, -1.0f);
    return make_float2(t1, t2);
}

// Train-time start jitter (reference raymarching.cu:195-198): only for rays that hit the box.
__device__ __forceinline__ float march_jitter(float t1, float noise, const MarchConst& c) {
    if (t1 >= 0.0f) t1 = __fmaf_rn(march_dt(t1, c), noise, t1);
    return t1;
}

// -------------------------------------------------------------------------------------------------
// One visit of the marcher at parameter t: the only place the per-point arithmetic is written. The serial
// visit below and the warp marcher (which probes 32 chain points at once) both use march_probe.
// -------------------------------------------------------------------------------------------------
struct MarchProbe {
    bool occ;
    float dt;        // step at this chain point (the sample's delta)
    float t_target;  // where an empty visit here jumps to (valid when !occ)
};

// One-entry cache of the occupancy lookup for a thread that marches one ray serially: consecutive samples of a ray fall
// into the same cell of the 128^3 grid ~4.6 times in a row (step 1/590 of the box diagonal vs cell 1/128), and the bit
// load is the one dependent global load on the visit's critical path. idx = 0xffffffff: empty.
struct MarchCache {
    uint32_t idx = 0xffffffffu;
    bool occ = false;
};

// ONE_CASCADE: with a single cascade both mip_from_pos and mip_from_dt clamp to 0 (min(cascades-1, .)), so
// mip = 0 and mip_bound = min(2^-1, scale) for every sample: the two frexpf, the scalbnf and the division drop out.
// With a cache the bit lookup is reused while the cell index is unchanged (same arithmetic, same roundings).
template <bool ONE_CASCADE>
__device__ __forceinline__ MarchProbe march_probe(const MarchRay& r, const MarchConst& c, float t,
                                                  MarchCache* cache = nullptr) {
    MarchProbe o;
    const float x = __fmaf_rn(r.dx, t, r.ox);
    const float y = __fmaf_rn(r.dy, t, r.oy);
    const float z = __fmaf_rn(r.dz, t, r.oz);
    o.dt = march_dt(t, c);
    int mip = 0;
    float mip_bound, mip_bound_inv;
    if (ONE_CASCADE) {
        mip_bound = c.mb0;
        mip_bound_inv = c.mb0_inv;
    } else {
        int e_pos, e_dt;
        frexpf(fmaxf(fabsf(x), fmaxf(fabsf(y), fabsf(z))), &e_pos);
        frexpf(__fmul_rn(o.dt, c.gs_f), &e_dt);
        mip = max(min(c.cascades - 1, max(0, e_pos + 1)), min(c.cascades - 1, max(0, e_dt)));
        mip_bound = fminf(scalbnf(1.0f, mip - 1), c.scale);
        mip_bound_inv = __fdiv_rn(1.0f, mip_bound);
    }
    const float vx = __fmul_rn(__fmul_rn(__fmaf_rn(x, mip_bound_inv, 1.0f), 0.5f), c.gs_f);
    const float vy = __fmul_rn(__fmul_rn(__fmaf_rn(y, mip_bound_inv, 1.0f), 0.5f), c.gs_f);
    const float vz = __fmul_rn(__fmul_rn(__fmaf_rn(z, mip_bound_inv, 1.0f), 0.5f), c.gs_f);
    const int nx = (int)fmaxf(0.0f, fminf(vx, c.gs_m1));
    const int ny = (int)fmaxf(0.0f, fminf(vy, c.gs_m1));
    const int nz = (int)fmaxf(0.0f, fminf(vz, c.gs_m1));
    const uint32_t idx = (uint32_t)mip * c.grid_size3 + morton_encode3((uint32_t)nx, (uint32_t)ny, (uint32_t)nz);
    if (!cache) {
        o.occ = (__ldg(c.bitfield + (idx >> 3)) >> (idx & 7u)) & 1u;
    } else {
        if (idx != cache->idx) {
            cache->occ = (__ldg(c.bitfield + (idx >> 3)) >> (idx & 7u)) & 1u;
            cache->idx = idx;
        }
        o.occ = cache->occ;
    }
    // distance to the exit face of this cell along each axis
    float a;
    a = __fmaf_rn(r.sx, 0.5f, __fadd_rn((float)nx, 0.5f));
    a = __fmaf_rn(__fmul_rn(a, c.gs_inv), 2.0f, -1.0f);
    const float tx = __fmul_rn(__fmaf_rn(mip_bound, a, -x), r.ix);
    a = __fmaf_rn(r.sy, 0.5f, __fadd_rn((float)ny, 0.5f));
    a = __fmaf_rn(__fmul_rn(a, c.gs_inv), 2.0f, -1.0f);
    const float ty = __fmul_rn(__fmaf_rn(mip_bound, a, -y), r.iy);
    a = __fmaf_rn(r.sz, 0.5f, __fadd_rn((float)nz, 0.5f));
    a = __fmaf_rn(__fmul_rn(a, c.gs_inv), 2.0f, -1.0f);
    const float tz = __fmul_rn(__fmaf_rn(mip_bound, a, -z), r.iz);
    o.t_target = __fadd_rn(t, fmaxf(0.0f, fminf(tx, fminf(ty, tz))));
    return o;
}

// Serial visit. Returns true when the cell under the ray is occupied (then dt is the sample's step, the sample sits at
// fma(d, t, o) and the caller advances t += dt); otherwise t has already been advanced past the empty cell, step by step
// like the reference. CONST_DT: the step is the constant dt_lo (see march_const_dt), the same value without the
// multiply and clamp.
template <bool CONST_DT, bool ONE_CASCADE>
__device__ __forceinline__ bool march_visit_t(const MarchRay& r, const MarchConst& c, float& t, float& dt,
                                              MarchCache* cache = nullptr) {
    const MarchProbe pr = march_probe<ONE_CASCADE>(r, c, t, cache);
    dt = pr.dt;
    if (pr.occ) return true;
    do {
        t = __fadd_rn(t, CONST_DT ? c.dt_lo : march_dt(t, c));
    } while (t < pr.t_target);
    return false;
}

// -------------------------------------------------------------------------------------------------
// Warp-cooperative marcher (one WARP per ray), bit-exact with the serial one.
//
// Every parameter value the reference ever visits lies on the ray's STEP CHAIN
//     c_0 = t_start,   c_{k+1} = c_k (+) dt(c_k)          ((+) = one fp32 rounded add)
// because both branches of its loop advance t the same way: an occupied visit does t += dt(t), an empty
// visit repeats t += dt(t) until t >= t_target. So the marcher is a walk over that chain: at a visited
// point test the cell; if occupied emit it and go to the next chain point, else jump to the first chain
// point >= t_target. Here a warp materialises 32 consecutive chain points (31 dependent rounded adds,
// identical roundings to the serial code), tests all 32 cells at once, and resolves which of them the
// serial walk would have visited with ballots. One thread per ray is latency bound (a dependent
// load + ~60 dependent ALU ops per visit, ~2 warps per SM at 8192 rays); this keeps the same
// sequence of fp32 operations per chain point but runs 32 of them side by side.
// -------------------------------------------------------------------------------------------------
// March one ray with a full warp. emit(k, t, dt) is called by the lane owning the k-th sample
// (k = 0.. in ray order). Returns the number of samples (same in every lane) and leaves in t_resume the
// chain point the serial marcher would visit next (what raymarching_test stores back into hits_t).
// CONST_DT: exp_step_factor == 0 (synthetic scenes): t*0 clamps to dt_lo for every finite t >= 0, so the step
// is the constant dt_lo and the chain needs one rounded add per point (same value, same rounding).
template <bool CONST_DT, bool ONE_CASCADE, class FEmit>
__device__ __forceinline__ int march_ray_warp(const MarchRay& ray, const MarchConst& c, float t_start, float t2,
                                              int max_new, int lane, FEmit emit, float* t_resume = nullptr) {
    int n = 0;
    float t = t_start;
    bool pending = false;   // an empty visit jumped past the end of the previous block
    float skip_to = 0.f;
    bool alive = (0.0f <= t) && (t < t2) && (max_new > 0);
    float resume = t_start;
    while (alive) {
        // 1. 32 consecutive chain points: lane j holds c_j
        float p = t;
        bool chain_done = false;
        if (CONST_DT) {
            // Inside one binade every rounded add of the constant step moves t by the same multiple of its ulp, so the
            // chain is t + j*inc with inc = fl(t + dt) - t (exact). Guess that, then CHECK the defining recurrence
            // c_j == fl(c_{j-1} + dt) in every lane; any mismatch (binade crossing, a tie) takes the serial adds below,
            // so the values are the serial ones bit for bit either way.
            const float inc = __fadd_rn(__fadd_rn(t, c.dt_lo), -t);
            const float guess = __fmaf_rn((float)lane, inc, t);
            const float prev = __shfl_up_sync(0xffffffffu, guess, 1);
            const bool ok = lane == 0 || __fadd_rn(prev, c.dt_lo) == guess;
            if (__all_sync(0xffffffffu, ok)) {
                p = guess;
                chain_done = true;
            }
        }
        if (!chain_done) {
#pragma unroll
            for (int j = 0; j < 31; ++j) {
                const float nx = __fadd_rn(p, CONST_DT ? c.dt_lo : march_dt(p, c));
                if (lane > j) p = nx;
            }
        }
        float t_next = __fadd_rn(p, CONST_DT ? c.dt_lo : march_dt(p, c));
        t_next = __shfl_sync(0xffffffffu, t_next, 31);
        // 2. probe all 32 cells
        const bool valid = p < t2;
        const MarchProbe pr = march_probe<ONE_CASCADE>(ray, c, p);
        const unsigned valid_mask = __ballot_sync(0xffffffffu, valid);
        const unsigned occ_mask = __ballot_sync(0xffffffffu, valid && pr.occ);
        // 3. which of them does the serial walk visit? An empty visit at lane j jumps to the first chain point that is not
        // below its t_target: every lane finds that successor for its own point with a binary search over the (increasing)
        // chain values, so the walk below costs one shuffle per empty visit.
        int nxt;
        {
            int lo = lane + 1, hi = 32;
#pragma unroll
            for (int it = 0; it < 5; ++it) {
                const int mid = (lo + hi) >> 1;
                const float pm = __shfl_sync(0xffffffffu, p, mid & 31);
                const bool ge = mid < 32 && !(pm < pr.t_target);
                if (lo < hi) {
                    if (ge) hi = mid;
                    else lo = mid + 1;
                }
            }
            nxt = lo;
        }
        int cur = 0;
        if (pending) {
            const unsigned m = __ballot_sync(0xffffffffu, !(p < skip_to));
            cur = m ? (__ffs(m) - 1) : 32;
            pending = (m == 0u);
        }
        unsigned sample_mask = 0u;
        // The walk is the orbit of `cur` under  succ(j) = 32 (j past the box: stop) | j+1 (occupied: a sample) | nxt_j (empty).
        // Pointer jumping gives the whole visited set in 5 rounds (one warp reduction + one shuffle each) instead of a
        // dependent iteration per visit.
        const int room0 = max_new - n;
        if (room0 > 32) {
            // more budget than points in the block: every visited occupied point is a sample
            unsigned visited = cur < 32 ? (1u << cur) : 0u;
            int jump = !valid ? 32 : (pr.occ ? lane + 1 : nxt);
#pragma unroll
            for (int r = 0; r < 5; ++r) {
                const unsigned contrib = (((visited >> lane) & 1u) && jump < 32) ? (1u << jump) : 0u;
                visited |= __reduce_or_sync(0xffffffffu, contrib);
                const int jj = __shfl_sync(0xffffffffu, jump, jump & 31);
                jump = jump < 32 ? jj : 32;
            }
            sample_mask = visited & occ_mask;
            const unsigned exits = visited & ~valid_mask;  // at most one: succ(invalid) stops the orbit
            if (exits) {  // t >= t2: the ray left the box
                alive = false;
                resume = __shfl_sync(0xffffffffu, p, __ffs(exits) - 1);
            } else if (visited) {
                // the last visited point: an empty one jumped past this block (carry its target over), an occupied one is
                // lane 31 and the walk simply continues with the next block
                const int last = 31 - __clz(visited);
                if (!((occ_mask >> last) & 1u)) {
                    pending = true;
                    skip_to = __shfl_sync(0xffffffffu, pr.t_target, last);
                }
            }
        } else
        while (cur < 32) {  // the budget may run out inside this block (test-time rounds, max_samples): the literal walk
            if (!((valid_mask >> cur) & 1u)) {  // t >= t2: the ray left the box
                alive = false;
                resume = __shfl_sync(0xffffffffu, p, cur);
                break;
            }
            const int room = max_new - n - __popc(sample_mask);
            if (room <= 0) {  // N_samples reached max_samples
                alive = false;
                resume = __shfl_sync(0xffffffffu, p, cur);
                break;
            }
            if ((occ_mask >> cur) & 1u) {
                // a run of occupied points: each is a sample and the next chain point is visited next
                const unsigned rest = (~occ_mask) >> cur;
                int run = rest ? (__ffs(rest) - 1) : (32 - cur);
                run = min(run, room);
                const unsigned bits = run >= 32 ? 0xffffffffu : ((1u << run) - 1u);
                sample_mask |= bits << cur;
                cur += run;
            } else {
                // empty cell: jump to the first chain point that is not below t_target
                const int to = __shfl_sync(0xffffffffu, nxt, cur);
                if (to >= 32) {  // past this block of 32: carry the target over
                    pending = true;
                    skip_to = __shfl_sync(0xffffffffu, pr.t_target, cur);
                }
                cur = to;
            }
        }
        if ((sample_mask >> lane) & 1u) emit(n + __popc(sample_mask & ((1u << lane) - 1u)), p, pr.dt);
        n += __popc(sample_mask);
        if (alive) {
            resume = t_next;
            t = t_next;
            if (!(t < t2)) alive = false;
        }
    }
    if (t_resume) *t_resume = resume;
    return n;
}

// -------------------------------------------------------------------------------------------------
// Host side: which specialisation of a marching kernel to launch.
// -------------------------------------------------------------------------------------------------
// The step is the constant dt_lo when exp_step_factor == 0 and dt_lo <= dt_hi: march_dt clamps t*0 up to dt_lo for every
// finite t >= 0. dt_scale is what make_march_const receives for dt_hi (the train kernel's scale, the test kernel's cascades).
inline bool march_const_dt(float esf, int max_samples, float dt_scale, int grid_size) {
    return esf == 0.0f && 1.73205080757f / (float)max_samples <= dt_scale * 3.46410161514f / (float)grid_size;
}

// Calls launch(std::integral_constant<bool, CONST_DT>{}, std::integral_constant<bool, ONE_CASCADE>{}) for the instance
// that serves (const_dt, cascades); the call site launches k<decltype(cd)::value, decltype(oc)::value>.
template <class Launch>
inline void march_dispatch(bool const_dt, int cascades, Launch&& launch) {
    using T = std::true_type;
    using F = std::false_type;
    if (const_dt && cascades == 1) launch(T{}, T{});
    else if (const_dt) launch(T{}, F{});
    else if (cascades == 1) launch(F{}, T{});
    else launch(F{}, F{});
}
