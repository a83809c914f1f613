// MSDA core forward for sm_90a -- sdetr_msda_forward / _ex / sdetr_msda_fused_forward.
//
// Reference semantics: models/bricks/ops/cuda/ms_deform_im2col_cuda.cuh:22-73,226-288 (kernel) and
// models/bricks/ms_deform_attn.py:322-344 (softmax + sampling-location arithmetic, fused variant).
//
// Design (not a port of the reference kernel, which maps one thread to one output scalar and issues
// 64 dependent 4-byte gathers per thread):
//   * a "group" of D/4 lanes owns one (image, query, head); every corner fetch is one 128-bit load per
//     lane, so a warp instruction moves four complete 128-byte head rows (D = 32);
//   * the 2*L*P sampling coordinates and L*P attention weights of the (query, head) are loaded ONCE,
//     coalesced, spread over the lanes of the group, and broadcast point by point with warp shuffles;
//   * in the fused variant the lanes run the L*P-way softmax with shuffle reductions and turn raw
//     offsets into sampling locations themselves, so neither tensor round-trips through HBM;
//   * the P points of a level are fetched together (4*P independent 128-bit loads in flight per lane);
//   * level shapes are read once per thread from the reference's int64 device tensors;
//   * queries may be processed in a caller-supplied (spatially tiled) order, either query-major
//     (all heads of 256/(8*M) consecutive queries per CTA) or head-major (one head of a chunk of
//     consecutive queries per CTA) so that co-resident groups gather from the same value neighbourhood
//     and hit in L1 instead of L2.  Output rows stay in the caller's order.
#include "msda.cuh"

namespace sdetr {

constexpr int kThreads = 256;

// ---- per-point setup, spread over the lanes of a group ----------------------------------------------------
// Point e (= level*P + point) of a (query, head) is owned by lane e % LANES, slot e / LANES.  The owner turns
// its sampling location into everything the gather needs -- top-left token index, two "has a neighbour" bits
// and the four corner weights (already multiplied by the attention weight, zero for corners outside the map)
// -- exactly once; the other lanes receive it with five shuffles instead of redoing ~50 instructions each.
struct LevelGeom {
    int H, W;
    float Hf, Wf;
    int64_t start;  // level_start_index
};

struct PointSetup {
    uint32_t packed;  // bits 0..29 token index (row-major) of the clamped top-left corner, bit 30 dx, bit 31 dy
    float w00, w01, w10, w11;
};

__device__ __forceinline__ PointSetup make_setup(float x, float y, float a, int H, int W, float Hf, float Wf) {
    PointSetup s;
    const float h_im = fmaf(y, Hf, -0.5f), w_im = fmaf(x, Wf, -0.5f);           // .cuh:274-275
    const bool in = h_im > -1.f && w_im > -1.f && h_im < Hf && w_im < Wf;        // .cuh:277
    const float hf = floorf(h_im), wf = floorf(w_im);
    const int y0 = (int)hf, x0 = (int)wf;
    const float ly = h_im - hf, lx = w_im - wf, hy = 1.f - ly, hx = 1.f - lx;
    const bool top = y0 >= 0, bot = y0 + 1 <= H - 1, lef = x0 >= 0, rig = x0 + 1 <= W - 1;
    // selected, not multiplied: a non-finite location (in == false, NaN fractions) contributes exactly 0 like the reference's
    // branch (.cuh:277) and like msda_backward.cu, instead of 0 * NaN
    s.w00 = (in && top && lef) ? a * hy * hx : 0.f;
    s.w01 = (in && top && rig) ? a * hy * lx : 0.f;
    s.w10 = (in && bot && lef) ? a * ly * hx : 0.f;
    s.w11 = (in && bot && rig) ? a * ly * lx : 0.f;
    // clamped corner rows/cols: every address is inside the level, invalid corners carry weight 0
    const int rt = max(y0, 0), rb = min(y0 + 1, H - 1), cl = max(x0, 0), cr = min(x0 + 1, W - 1);
    const uint32_t idx = (uint32_t)(rt * W + cl), dx = (uint32_t)(cr - cl), dy = (uint32_t)(rb - rt);
    s.packed = in ? (idx | (dx << 30) | (dy << 31)) : 0u;
    return s;
}

// address = base + index * stride_bytes in ONE mad.wide.u32
__device__ __forceinline__ const float *row_ptr(const char *base, uint32_t index, uint32_t stride_bytes) {
    uint64_t r;
    asm("mad.wide.u32 %0, %1, %2, %3;" : "=l"(r) : "r"(index), "r"(stride_bytes), "l"(reinterpret_cast<uint64_t>(base)));
    return reinterpret_cast<const float *>(r);
}

__device__ __forceinline__ void fma4(float4 &acc, float w, const float4 &v) {
    acc.x = fmaf(w, v.x, acc.x), acc.y = fmaf(w, v.y, acc.y), acc.z = fmaf(w, v.z, acc.z), acc.w = fmaf(w, v.w, acc.w);
}

// gather of one level: the P points are fetched together (4*P independent 128-bit loads per lane).
// Addresses are base64 + token_index * stride with ONE IMAD.WIDE.U32 each (32-bit index and stride).
template <int L, int P, int LANES, int SLOTS, int LVL = 0>
struct LevelLoop {
    static __device__ __forceinline__ void run(float4 &acc, const PointSetup (&st)[SLOTS], const LevelGeom (&geo)[L],
                                               const float *__restrict__ vbase, uint32_t ts) {
        // byte arithmetic on purpose: address = 64-bit level base + (32-bit token index) * (32-bit byte stride)
        const char *lvl_base = reinterpret_cast<const char *>(vbase + geo[LVL].start * (int64_t)ts);
        const uint32_t tsb = ts * 4u;
        const uint32_t W = (uint32_t)geo[LVL].W;
        float4 v[P][4];
        float w[P][4];
#pragma unroll
        for (int pt = 0; pt < P; ++pt) {
            const int e = LVL * P + pt;  // compile-time after unrolling
            const int src = e % LANES, slot = e / LANES;
            const uint32_t pk = __shfl_sync(0xffffffffu, st[slot].packed, src, LANES);
            w[pt][0] = __shfl_sync(0xffffffffu, st[slot].w00, src, LANES);
            w[pt][1] = __shfl_sync(0xffffffffu, st[slot].w01, src, LANES);
            w[pt][2] = __shfl_sync(0xffffffffu, st[slot].w10, src, LANES);
            w[pt][3] = __shfl_sync(0xffffffffu, st[slot].w11, src, LANES);
            const uint32_t i00 = pk & 0x3fffffffu;
            const uint32_t i01 = i00 + ((pk >> 30) & 1u);
            const uint32_t i10 = i00 + (pk >> 31) * W;
            const uint32_t i11 = i10 + ((pk >> 30) & 1u);
            v[pt][0] = ldg_f4(row_ptr(lvl_base, i00, tsb));
            v[pt][1] = ldg_f4(row_ptr(lvl_base, i01, tsb));
            v[pt][2] = ldg_f4(row_ptr(lvl_base, i10, tsb));
            v[pt][3] = ldg_f4(row_ptr(lvl_base, i11, tsb));
        }
#pragma unroll
        for (int pt = 0; pt < P; ++pt) {
#pragma unroll
            for (int c = 0; c < 4; ++c) fma4(acc, w[pt][c], v[pt][c]);
        }
        if constexpr (LVL + 1 < L) LevelLoop<L, P, LANES, SLOTS, LVL + 1>::run(acc, st, geo, vbase, ts);
    }
};

// Variant B of the gather: the owners publish their setups in shared memory (one STS.128 + one STS.32 per
// point) and every lane reads a level's four packed indices with ONE LDS.128 and each point's four weights with
// ONE LDS.128 (warp-wide broadcast reads: 4 distinct 16-byte chunks in distinct banks) -- 5 shared-memory
// wavefronts per level instead of 20 shuffle wavefronts on the same LSU data pipe that the gathers saturate.
constexpr int kWStride = 336;  // bytes per group for weights: 16 points x 16 B, padded so 4 groups hit distinct banks
constexpr int kPkStride = 80;  // bytes per group for packed indices: 16 x 4 B, padded likewise

template <int L, int P, int LANES, int LVL = 0>
struct LevelLoopSmem {
    static __device__ __forceinline__ void run(float4 &acc, const char *wsm, const char *pksm, const LevelGeom (&geo)[L],
                                               const float *__restrict__ vbase, uint32_t ts) {
        static_assert(P == 4, "one LDS.128 carries the four packed indices of a level");
        const char *lvl_base = reinterpret_cast<const char *>(vbase + geo[LVL].start * (int64_t)ts);
        const uint32_t tsb = ts * 4u;
        const uint32_t W = (uint32_t)geo[LVL].W;
        const uint4 pk4 = *reinterpret_cast<const uint4 *>(pksm + LVL * 16);
        const uint32_t pks[4] = {pk4.x, pk4.y, pk4.z, pk4.w};
        float4 v[P][4], w[P];
#pragma unroll
        for (int pt = 0; pt < P; ++pt) {
            w[pt] = *reinterpret_cast<const float4 *>(wsm + (LVL * P + pt) * 16);
            const uint32_t pk = pks[pt];
            const uint32_t i00 = pk & 0x3fffffffu;
            const uint32_t i01 = i00 + ((pk >> 30) & 1u);
            const uint32_t i10 = i00 + (pk >> 31) * W;
            const uint32_t i11 = i10 + ((pk >> 30) & 1u);
            v[pt][0] = ldg_f4(row_ptr(lvl_base, i00, tsb));
            v[pt][1] = ldg_f4(row_ptr(lvl_base, i01, tsb));
            v[pt][2] = ldg_f4(row_ptr(lvl_base, i10, tsb));
            v[pt][3] = ldg_f4(row_ptr(lvl_base, i11, tsb));
        }
#pragma unroll
        for (int pt = 0; pt < P; ++pt) {
            fma4(acc, w[pt].x, v[pt][0]);
            fma4(acc, w[pt].y, v[pt][1]);
            fma4(acc, w[pt].z, v[pt][2]);
            fma4(acc, w[pt].w, v[pt][3]);
        }
        if constexpr (LVL + 1 < L) LevelLoopSmem<L, P, LANES, LVL + 1>::run(acc, wsm, pksm, geo, vbase, ts);
    }
};

// level geometry of the point owned by (slot, lane): only the levels a slot can span are tested
template <int L, int P, int LANES, int SLOT>
__device__ __forceinline__ void slot_geom(const LevelGeom (&geo)[L], int lane, int &l, int &H, int &W, float &Hf, float &Wf) {
    constexpr int lo = (SLOT * LANES) / P < L - 1 ? (SLOT * LANES) / P : L - 1;
    constexpr int hi = (SLOT * LANES + LANES - 1) / P < L - 1 ? (SLOT * LANES + LANES - 1) / P : L - 1;
    const int e = SLOT * LANES + lane;
    l = min(e / P, L - 1);
    H = geo[lo].H, W = geo[lo].W, Hf = geo[lo].Hf, Wf = geo[lo].Wf;
#pragma unroll
    for (int k = lo + 1; k <= hi; ++k)
        if (l == k) H = geo[k].H, W = geo[k].W, Hf = geo[k].Hf, Wf = geo[k].Wf;
}

template <int L, int P, int LANES, int SLOTS, bool FUSED, int SLOT = 0>
struct SlotLoop {
    // FUSED: (lx, ly) raw offsets -> locations (needs ref), la normalised; then the setup of every slot
    static __device__ __forceinline__ void run(PointSetup (&st)[SLOTS], float (&lx)[SLOTS], float (&ly)[SLOTS],
                                               float (&la)[SLOTS], const LevelGeom (&geo)[L], int lane,
                                               const float *__restrict__ rrow, float inv_sum, int ref_dim) {
        int l, H, W;
        float Hf, Wf;
        slot_geom<L, P, LANES, SLOT>(geo, lane, l, H, W, Hf, Wf);
        if constexpr (FUSED) {
            fused_location<P>(rrow, l, ref_dim, lx[SLOT], ly[SLOT], Wf, Hf, lx[SLOT], ly[SLOT]);
            la[SLOT] = la[SLOT] * inv_sum;
        }
        st[SLOT] = make_setup(lx[SLOT], ly[SLOT], la[SLOT], H, W, Hf, Wf);
        if constexpr (SLOT + 1 < SLOTS)
            SlotLoop<L, P, LANES, SLOTS, FUSED, SLOT + 1>::run(st, lx, ly, la, geo, lane, rrow, inv_sum, ref_dim);
    }
};

// ---- the specialised kernel -------------------------------------------------------------------------
template <int D, int L, int P, bool FUSED, bool HEAD_MAJOR, int MINB, bool SMEM_BCAST = false, int THREADS = kThreads>
__global__ void __launch_bounds__(THREADS, MINB) msda_fwd_kernel(const MsdaFwdParams p) {
    constexpr int LANES = D / 4;
    constexpr int GROUPS = THREADS / LANES;
    constexpr int NP = L * P;
    constexpr int SLOTS = (NP + LANES - 1) / LANES;
    const int lane = threadIdx.x % LANES;
    const int grp = threadIdx.x / LANES;

    LevelGeom geo[L];
#pragma unroll
    for (int l = 0; l < L; ++l) {
        geo[l].H = (int)__ldg(p.shapes + 2 * l);
        geo[l].W = (int)__ldg(p.shapes + 2 * l + 1);
        geo[l].Hf = (float)geo[l].H, geo[l].Wf = (float)geo[l].W;
        geo[l].start = __ldg(p.lsi + l);
    }

    // Work assignment.  Every lane of a warp runs the same number of iterations (the shuffles below
    // use the full mask); out-of-range groups recompute a valid item and skip the store.
    int b, m, q_first, q_last, q_step, iters;
    bool in_range = true;
    if constexpr (HEAD_MAJOR) {
        b = blockIdx.z, m = blockIdx.y;
        q_first = blockIdx.x * p.chunk + grp;
        q_last = min(p.nq, (int)(blockIdx.x + 1) * p.chunk) - 1;  // >= blockIdx.x*chunk by construction
        q_step = GROUPS;
        iters = (p.chunk + GROUPS - 1) / GROUPS;
    } else {
        b = blockIdx.y;
        uint32_t item = blockIdx.x * GROUPS + grp;  // (query, head) of this image
        in_range = item < (uint32_t)p.nq * (uint32_t)p.heads;
        if (!in_range) item = 0;
        q_first = q_last = (int)(item / (uint32_t)p.heads);
        m = (int)(item - (uint32_t)q_first * (uint32_t)p.heads);
        q_step = 0;
        iters = 1;
    }

    for (int it = 0; it < iters; ++it) {
        int qi = q_first + it * q_step;
        const bool active = in_range && qi <= q_last;
        qi = min(qi, q_last);
        const int q = p.order ? __ldg(p.order + (int64_t)b * p.nq + qi) : qi;
        const int64_t row = (int64_t)b * p.nq + q;  // (image, query) row of every per-query tensor
        const int64_t qm = row * p.heads + m;

        // ---- phase 1: each lane prepares its own points -----------------------------------------------------
        float lx[SLOTS], ly[SLOTS], la[SLOTS];
        float inv_sum = 1.f;
        const float *rrow = nullptr;
        if constexpr (FUSED) {
            const float *prow = p.proj + row * p.proj_stride;
            const float *offs = prow + (int64_t)m * 2 * NP;                      // raw offsets of this head
            const float *logit = prow + (int64_t)p.heads * 2 * NP + (int64_t)m * NP;  // raw logits of this head
            float mx = -INFINITY;
#pragma unroll
            for (int s = 0; s < SLOTS; ++s) {
                const int e = s * LANES + lane;
                const bool ok = (NP % LANES == 0) || e < NP;
                const float2 o = ok ? __ldg(reinterpret_cast<const float2 *>(offs) + e) : make_float2(0.f, 0.f);
                lx[s] = o.x, ly[s] = o.y;
                la[s] = ok ? __ldg(logit + e) : -INFINITY;
                mx = fmaxf(mx, la[s]);
            }
            mx = group_max<LANES>(mx);  // softmax over the L*P logits (ms_deform_attn.py:326-329)
            float sum = 0.f;
#pragma unroll
            for (int s = 0; s < SLOTS; ++s) la[s] = __expf(la[s] - mx), sum += la[s];
            sum = group_sum<LANES>(sum);
            inv_sum = __frcp_rn(sum);
            rrow = p.ref + row * (p.ref_dim * L);
        } else {
#pragma unroll
            for (int s = 0; s < SLOTS; ++s) {
                const int e = s * LANES + lane;
                const bool ok = (NP % LANES == 0) || e < NP;
                const float2 o = ok ? __ldg(reinterpret_cast<const float2 *>(p.loc + qm * (2 * NP)) + e) : make_float2(0.f, 0.f);
                lx[s] = o.x, ly[s] = o.y;
                la[s] = ok ? __ldg(p.attn + qm * NP + e) : 0.f;
            }
        }
        PointSetup st[SLOTS];
        SlotLoop<L, P, LANES, SLOTS, FUSED>::run(st, lx, ly, la, geo, lane, rrow, inv_sum, p.ref_dim);
        if constexpr (FUSED) {
            if (active) {
#pragma unroll
                for (int s = 0; s < SLOTS; ++s) {
                    const int e = s * LANES + lane;
                    if ((NP % LANES == 0) || e < NP) {
                        if (p.loc_out) reinterpret_cast<float2 *>(p.loc_out + qm * (2 * NP))[e] = make_float2(lx[s], ly[s]);
                        if (p.attn_out) p.attn_out[qm * NP + e] = la[s];
                    }
                }
            }
        }

        // ---- phase 2: gather ------------------------------------------------------------------------------------
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        const float *vbase = p.value + (int64_t)b * p.v_bstride + (int64_t)m * D + lane * 4;
        if constexpr (SMEM_BCAST) {
            static_assert(!SMEM_BCAST || (NP == 16 && LANES == 8), "shared-memory broadcast variant: 16 points, 8 lanes");
            extern __shared__ __align__(16) char bc_smem[];  // GROUPS * (kWStride + kPkStride) bytes (dynamic)
            char *wsm = bc_smem + grp * kWStride;
            char *pksm = bc_smem + GROUPS * kWStride + grp * kPkStride;
#pragma unroll
            for (int s = 0; s < SLOTS; ++s) {
                const int e = s * LANES + lane;
                *reinterpret_cast<float4 *>(wsm + e * 16) = make_float4(st[s].w00, st[s].w01, st[s].w10, st[s].w11);
                *reinterpret_cast<uint32_t *>(pksm + e * 4) = st[s].packed;
            }
            __syncwarp();
            LevelLoopSmem<L, P, LANES>::run(acc, wsm, pksm, geo, vbase, (uint32_t)p.v_tstride);
            __syncwarp();  // all lanes have read this item's setups before the next item overwrites them
        } else {
            LevelLoop<L, P, LANES, SLOTS>::run(acc, st, geo, vbase, (uint32_t)p.v_tstride);
        }
        if (active) st_stream_f4(p.out + qm * D + lane * 4, acc);
    }
}

// ---- "W32": one WARP per (image, query, head), one lane per channel (D = 32, L = 4, P = 4, head-major schedule) ------------
// The kernel above issues LDG.128 instructions that touch four different 128-byte lines each (one per 8-lane group), and a
// multi-line request is replayed line by line in the L1 tag stage, so even all-hit gathers cost more than their 128 B per row
// of data movement.  Here every corner row is ONE fully
// coalesced 128-byte LDG.32 -- a single line, a single wavefront -- issued by the whole warp:
//   * lane e (and its mirror e + 16) owns sampling point e of the (query, head): softmax over 16 lanes by shuffles,
//     location, corner index and the four weights are computed once per point and published in 320 bytes of shared memory
//     per warp; every lane then reads a level's four indices with one uniform LDS.128 and each point's weights with one
//     uniform LDS.128 (1 wavefront each: 20 per item instead of 80 shuffles);
//   * 16 (one level) or 32 (two levels) independent corner loads in flight per lane, one FMA each; ~40 registers, so up
//     to 48 warps per SM;
//   * the 8 warps of a CTA walk consecutive queries of the tile order (same head), so co-resident gathers share lines.
constexpr int kW32Warps = 8;

template <bool FUSED, int LVB /* levels gathered per batch: 1 or 2 */, int MINB>
__global__ void __launch_bounds__(kW32Warps * 32, MINB) msda_fwd_w32_kernel(const MsdaFwdParams p) {
    constexpr int L = 4, P = 4, NP = 16, D = 32;
    __shared__ __align__(16) float4 s_w[kW32Warps][NP];
    __shared__ __align__(16) uint32_t s_pk[kW32Warps][NP];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, e = lane & 15, lvl_e = e >> 2;
    LevelGeom geo[L];
#pragma unroll
    for (int l = 0; l < L; ++l) {
        geo[l].H = (int)__ldg(p.shapes + 2 * l);
        geo[l].W = (int)__ldg(p.shapes + 2 * l + 1);
        geo[l].Hf = (float)geo[l].H, geo[l].Wf = (float)geo[l].W;
        geo[l].start = __ldg(p.lsi + l);
    }
    // geometry of the level this lane's point belongs to
    int He = geo[0].H, We = geo[0].W;
    float Hfe = geo[0].Hf, Wfe = geo[0].Wf;
#pragma unroll
    for (int l = 1; l < L; ++l)
        if (lvl_e == l) He = geo[l].H, We = geo[l].W, Hfe = geo[l].Hf, Wfe = geo[l].Wf;
    const int b = blockIdx.z, m = blockIdx.y;
    const int q_end = min(p.nq, (int)(blockIdx.x + 1) * p.chunk);
    const uint32_t tsb = (uint32_t)p.v_tstride * 4u;
    const char *vhead = reinterpret_cast<const char *>(p.value + (int64_t)b * p.v_bstride + (int64_t)m * D + lane);
    const char *lvl_base[L];
#pragma unroll
    for (int l = 0; l < L; ++l) lvl_base[l] = vhead + geo[l].start * (int64_t)tsb;

    for (int qi = blockIdx.x * p.chunk + warp; qi < q_end; qi += kW32Warps) {  // warp-uniform trip count
        const int q = p.order ? __ldg(p.order + (int64_t)b * p.nq + qi) : qi;
        const int64_t row = (int64_t)b * p.nq + q;
        const int64_t qm = row * p.heads + m;
        float x, y, a;
        if constexpr (FUSED) {
            const float *prow = p.proj + row * p.proj_stride;
            const float2 o = __ldg(reinterpret_cast<const float2 *>(prow + (int64_t)m * 2 * NP) + e);
            const float lg = __ldg(prow + (int64_t)p.heads * 2 * NP + (int64_t)m * NP + e);
            const float mx = group_max<16>(lg);  // softmax over the 16 logits (ms_deform_attn.py:326-329)
            const float ex = __expf(lg - mx);
            const float inv = __frcp_rn(group_sum<16>(ex));
            fused_location<P>(p.ref + row * (p.ref_dim * L), lvl_e, p.ref_dim, o.x, o.y, Wfe, Hfe, x, y);
            a = ex * inv;
            if (lane < NP) {
                if (p.loc_out) reinterpret_cast<float2 *>(p.loc_out + qm * (2 * NP))[e] = make_float2(x, y);
                if (p.attn_out) p.attn_out[qm * NP + e] = a;
            }
        } else {
            const float2 o = __ldg(reinterpret_cast<const float2 *>(p.loc + qm * (2 * NP)) + e);
            x = o.x, y = o.y;
            a = __ldg(p.attn + qm * NP + e);
        }
        const PointSetup st = make_setup(x, y, a, He, We, Hfe, Wfe);
        if (lane < NP) {
            s_w[warp][e] = make_float4(st.w00, st.w01, st.w10, st.w11);
            s_pk[warp][e] = st.packed;
        }
        __syncwarp();
        float acc = 0.f;
#pragma unroll
        for (int l0 = 0; l0 < L; l0 += LVB) {
            float v[LVB][P][4];
            float4 w[LVB][P];
#pragma unroll
            for (int dl = 0; dl < LVB; ++dl) {
                const int l = l0 + dl;
                const uint4 pk4 = *reinterpret_cast<const uint4 *>(&s_pk[warp][l * P]);
                const uint32_t pks[4] = {pk4.x, pk4.y, pk4.z, pk4.w};
                const uint32_t W = (uint32_t)geo[l].W;
#pragma unroll
                for (int pt = 0; pt < P; ++pt) {
                    w[dl][pt] = s_w[warp][l * P + pt];
                    const uint32_t pk = pks[pt];
                    const uint32_t i00 = pk & 0x3fffffffu;
                    const uint32_t i01 = i00 + ((pk >> 30) & 1u);
                    const uint32_t i10 = i00 + (pk >> 31) * W;
                    const uint32_t i11 = i10 + ((pk >> 30) & 1u);
                    v[dl][pt][0] = __ldg(row_ptr(lvl_base[l], i00, tsb));
                    v[dl][pt][1] = __ldg(row_ptr(lvl_base[l], i01, tsb));
                    v[dl][pt][2] = __ldg(row_ptr(lvl_base[l], i10, tsb));
                    v[dl][pt][3] = __ldg(row_ptr(lvl_base[l], i11, tsb));
                }
            }
#pragma unroll
            for (int dl = 0; dl < LVB; ++dl)
#pragma unroll
                for (int pt = 0; pt < P; ++pt) {
                    acc = fmaf(w[dl][pt].x, v[dl][pt][0], acc);
                    acc = fmaf(w[dl][pt].y, v[dl][pt][1], acc);
                    acc = fmaf(w[dl][pt].z, v[dl][pt][2], acc);
                    acc = fmaf(w[dl][pt].w, v[dl][pt][3], acc);
                }
        }
        __syncwarp();  // all lanes have read this item's setups before the next item overwrites them
        asm volatile("st.global.L1::no_allocate.f32 [%0], %1;" ::"l"(p.out + qm * D + lane), "f"(acc) : "memory");
    }
}

// ---- generic fallback (any head_dim % 4 == 0, L <= kMaxLevels, any P) ------------------------------------
__global__ void __launch_bounds__(kThreads) msda_fwd_generic_kernel(const MsdaFwdParams p, int D, int L, int P,
                                                                   int fused) {
    const int lanes = D / 4;
    const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = (int)(gid % lanes);
    const int64_t item = gid / lanes;
    const int m = (int)(item % p.heads);
    const int64_t bq = item / p.heads;
    const int qi = (int)(bq % p.nq);
    const int b = (int)(bq / p.nq);
    if (b >= p.batch) return;
    const int q = p.order ? __ldg(p.order + (int64_t)b * p.nq + qi) : qi;
    const int64_t row = (int64_t)b * p.nq + q;
    const int NP = L * P;
    const float *prow = fused ? p.proj + row * p.proj_stride : nullptr;
    float mx = -INFINITY, sum = 0.f;
    if (fused) {
        const float *lg = prow + (int64_t)p.heads * 2 * NP + (int64_t)m * NP;
        for (int i = 0; i < NP; ++i) mx = fmaxf(mx, __ldg(lg + i));
        for (int i = 0; i < NP; ++i) sum += expf(__ldg(lg + i) - mx);
    }
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    const float *vbase = p.value + (int64_t)b * p.v_bstride + (int64_t)m * D + lane * 4;
    for (int l = 0; l < L; ++l) {
        LevelGeom g;
        g.H = (int)__ldg(p.shapes + 2 * l), g.W = (int)__ldg(p.shapes + 2 * l + 1);
        g.Hf = (float)g.H, g.Wf = (float)g.W, g.start = __ldg(p.lsi + l);
        const float *lvl_base = vbase + g.start * p.v_tstride;
        for (int pt = 0; pt < P; ++pt) {
            const int e = l * P + pt;
            float x, y, a;
            if (fused) {
                const float *off = prow + (int64_t)m * 2 * NP + 2 * e;
                const float *rr = p.ref + row * (p.ref_dim * L) + p.ref_dim * l;
                if (p.ref_dim == 2) {
                    x = __ldg(rr) + __ldg(off) / g.Wf;
                    y = __ldg(rr + 1) + __ldg(off + 1) / g.Hf;
                } else {
                    x = __ldg(rr) + __fmul_rn(__fmul_rn(__fdiv_rn(__ldg(off), (float)P), __ldg(rr + 2)), 0.5f);
                    y = __ldg(rr + 1) + __fmul_rn(__fmul_rn(__fdiv_rn(__ldg(off + 1), (float)P), __ldg(rr + 3)), 0.5f);
                }
                a = expf(__ldg(prow + (int64_t)p.heads * 2 * NP + (int64_t)m * NP + e) - mx) / sum;
                if (lane == 0) {
                    if (p.loc_out) {
                        p.loc_out[((row * p.heads + m) * NP + e) * 2] = x;
                        p.loc_out[((row * p.heads + m) * NP + e) * 2 + 1] = y;
                    }
                    if (p.attn_out) p.attn_out[(row * p.heads + m) * NP + e] = a;
                }
            } else {
                const float *lp = p.loc + ((row * p.heads + m) * NP + e) * 2;
                x = __ldg(lp), y = __ldg(lp + 1);
                a = __ldg(p.attn + (row * p.heads + m) * NP + e);
            }
            const PointSetup st = make_setup(x, y, a, g.H, g.W, g.Hf, g.Wf);
            const float *p00 = lvl_base + (int64_t)(st.packed & 0x3fffffffu) * p.v_tstride;
            const int64_t dx = (st.packed & 0x40000000u) ? p.v_tstride : 0;
            const int64_t dy = (st.packed & 0x80000000u) ? (int64_t)g.W * p.v_tstride : 0;
            fma4(acc, st.w00, ldg_f4(p00));
            fma4(acc, st.w01, ldg_f4(p00 + dx));
            fma4(acc, st.w10, ldg_f4(p00 + dy));
            fma4(acc, st.w11, ldg_f4(p00 + dy + dx));
        }
    }
    *reinterpret_cast<float4 *>(p.out + (row * p.heads + m) * D + lane * 4) = acc;
}

// ---- host side -----------------------------------------------------------------------------------------
static std::atomic<int> g_bcast{1};  // 0 = shuffle broadcast, 1 = shared-memory broadcast (D=32, L=4, P=4 only)
static std::atomic<int> g_minb{4};   // tuning knobs (sdetr_set_option)
static std::atomic<int> g_chunk{64};
static std::atomic<int> g_threads{256};
int g_msda_host_shapes[2 * kMaxLevels + 1] = {0};  // [L, H_0, W_0, H_1, W_1, ...] for the TMA variant's tensor maps
static std::atomic<int> g_tma{0};      // head-major schedule, D=32/L=4/P=4: 1 = TMA-staged shared-memory windows (msda_forward_tma.cu)
static std::atomic<int> g_w32{0};      // head-major schedule, D=32/L=4/P=4: 0 = 8-lane groups (above), 1 / 2 = warp per item, 1 / 2 levels per batch  // head-major schedule: threads per CTA (256 x 4 CTAs/SM, 512 x 2, 1024 x 1)

template <int D, int L, int P, int MINB>
static void launch_special(const MsdaFwdParams &p, bool fused, int schedule, cudaStream_t s) {
    constexpr int GROUPS = kThreads / (D / 4);
    if (schedule == 1) {
        dim3 grid((p.nq + p.chunk - 1) / p.chunk, p.heads, p.batch);
        if (fused)
            msda_fwd_kernel<D, L, P, true, true, MINB><<<grid, kThreads, 0, s>>>(p);
        else
            msda_fwd_kernel<D, L, P, false, true, MINB><<<grid, kThreads, 0, s>>>(p);
    } else {
        const int64_t items = (int64_t)p.nq * p.heads;
        dim3 grid((unsigned)((items + GROUPS - 1) / GROUPS), p.batch);
        if (fused)
            msda_fwd_kernel<D, L, P, true, false, MINB><<<grid, kThreads, 0, s>>>(p);
        else
            msda_fwd_kernel<D, L, P, false, false, MINB><<<grid, kThreads, 0, s>>>(p);
    }
}

static int msda_forward_dispatch(MsdaFwdParams p, bool fused, int head_dim, int levels, int points, int schedule,
                                 cudaStream_t s) {
    SDETR_REQUIRE(p.nq >= 0, SDETR_ERR_INVALID_ARG, "msda_forward: negative num_query");
    if (p.nq == 0) return SDETR_OK;  // empty query set: nothing to do (empty tensors have null data pointers)
    SDETR_REQUIRE(p.value && p.shapes && p.lsi && p.out, SDETR_ERR_INVALID_ARG, "msda_forward: null pointer");
    SDETR_REQUIRE(fused ? (p.ref && p.proj) : (p.loc && p.attn), SDETR_ERR_INVALID_ARG,
                  "msda_forward: null sampling input");
    SDETR_REQUIRE(p.batch > 0 && p.nv > 0 && p.heads > 0 && levels > 0 && points > 0 && p.nq >= 0,
                  SDETR_ERR_INVALID_ARG, "msda_forward: non-positive size");
    SDETR_REQUIRE(head_dim % 4 == 0 && head_dim >= 4 && head_dim <= 1024, SDETR_ERR_UNSUPPORTED,
                  "msda_forward: head_dim %d must be a multiple of 4 (128-bit rows)", head_dim);
    SDETR_REQUIRE(levels <= kMaxLevels, SDETR_ERR_UNSUPPORTED, "msda_forward: more than %d levels", kMaxLevels);
    SDETR_REQUIRE(aligned16(p.value) && aligned16(p.out) && p.v_tstride % 4 == 0 && p.v_bstride % 4 == 0,
                  SDETR_ERR_INVALID_ARG, "msda_forward: value/output must be 16-byte aligned");
    SDETR_REQUIRE(schedule == 0 || schedule == 1, SDETR_ERR_INVALID_ARG, "msda_forward: bad schedule %d", schedule);
    p.chunk = g_chunk;
    SDETR_REQUIRE(p.batch <= 65535, SDETR_ERR_UNSUPPORTED, "msda_forward: batch > 65535");
    bool special = true;
    if (fused) special = (p.proj_stride % 4 == 0) && aligned16(p.proj);
    else special = aligned16(p.loc) && aligned16(p.attn);
    if (special && head_dim == 32 && levels == 4 && points == 4 && schedule == 1 && g_tma.load() != 0 && p.order) {
        return launch_msda_tma(p, fused, s);
    } else if (special && head_dim == 32 && levels == 4 && points == 4 && schedule == 1 && g_w32.load() != 0) {
        dim3 grid((p.nq + p.chunk - 1) / p.chunk, p.heads, p.batch);
        const int k = g_w32.load();
        if (k == 2) {
            if (fused) msda_fwd_w32_kernel<true, 2, 4><<<grid, kW32Warps * 32, 0, s>>>(p);
            else msda_fwd_w32_kernel<false, 2, 4><<<grid, kW32Warps * 32, 0, s>>>(p);
        } else {
            if (fused) msda_fwd_w32_kernel<true, 1, 6><<<grid, kW32Warps * 32, 0, s>>>(p);
            else msda_fwd_w32_kernel<false, 1, 6><<<grid, kW32Warps * 32, 0, s>>>(p);
        }
    } else if (special && head_dim == 32 && levels == 4 && points == 4 && g_bcast == 1) {
        const int threads = schedule == 1 ? g_threads.load() : kThreads;
        const int groups = threads / 8;
        const size_t smem = (size_t)groups * (kWStride + kPkStride);
        if (schedule == 1) {
            dim3 grid((p.nq + p.chunk - 1) / p.chunk, p.heads, p.batch);
            if (threads == 1024) {
                static PerDeviceOnce o1, o2;
                SDETR_OPT_IN_SMEM(o1, (msda_fwd_kernel<32, 4, 4, true, true, 1, true, 1024>), smem, "msda_forward");
                SDETR_OPT_IN_SMEM(o2, (msda_fwd_kernel<32, 4, 4, false, true, 1, true, 1024>), smem, "msda_forward");
                if (fused) msda_fwd_kernel<32, 4, 4, true, true, 1, true, 1024><<<grid, 1024, smem, s>>>(p);
                else msda_fwd_kernel<32, 4, 4, false, true, 1, true, 1024><<<grid, 1024, smem, s>>>(p);
            } else if (threads == 512) {
                if (fused) msda_fwd_kernel<32, 4, 4, true, true, 2, true, 512><<<grid, 512, smem, s>>>(p);
                else msda_fwd_kernel<32, 4, 4, false, true, 2, true, 512><<<grid, 512, smem, s>>>(p);
            } else {
                if (fused) msda_fwd_kernel<32, 4, 4, true, true, 4, true><<<grid, kThreads, smem, s>>>(p);
                else msda_fwd_kernel<32, 4, 4, false, true, 4, true><<<grid, kThreads, smem, s>>>(p);
            }
        } else {
            dim3 grid((unsigned)(((int64_t)p.nq * p.heads + groups - 1) / groups), p.batch);
            if (fused) msda_fwd_kernel<32, 4, 4, true, false, 4, true><<<grid, kThreads, smem, s>>>(p);
            else msda_fwd_kernel<32, 4, 4, false, false, 4, true><<<grid, kThreads, smem, s>>>(p);
        }
    } else if (special && head_dim == 32 && levels == 4 && points == 4) {
        if (g_minb == 3) launch_special<32, 4, 4, 3>(p, fused, schedule, s);
        else if (g_minb == 4) launch_special<32, 4, 4, 4>(p, fused, schedule, s);
        else if (g_minb == 5) launch_special<32, 4, 4, 5>(p, fused, schedule, s);
        else if (g_minb == 6) launch_special<32, 4, 4, 6>(p, fused, schedule, s);
        else launch_special<32, 4, 4, 2>(p, fused, schedule, s);
    } else if (special && head_dim == 32 && levels == 5 && points == 4)
        launch_special<32, 5, 4, 2>(p, fused, schedule, s);
    else if (special && head_dim == 64 && levels == 4 && points == 4)
        launch_special<64, 4, 4, 2>(p, fused, schedule, s);
    else {
        const int64_t threads = (int64_t)p.batch * p.nq * p.heads * (head_dim / 4);
        msda_fwd_generic_kernel<<<(unsigned)((threads + kThreads - 1) / kThreads), kThreads, 0, s>>>(
            p, head_dim, levels, points, fused ? 1 : 0);
    }
    return check_launch("msda_forward");
}

}  // namespace sdetr

using namespace sdetr;

extern "C" int sdetr_msda_set_host_shapes(int num_levels, const int32_t *level_h_host, const int32_t *level_w_host) {
    SDETR_REQUIRE(num_levels >= 0 && num_levels <= kMaxLevels && (num_levels == 0 || (level_h_host && level_w_host)),
                  SDETR_ERR_INVALID_ARG, "msda_set_host_shapes: bad arguments");
    g_msda_host_shapes[0] = num_levels;
    for (int l = 0; l < num_levels; ++l) g_msda_host_shapes[1 + 2 * l] = level_h_host[l], g_msda_host_shapes[2 + 2 * l] = level_w_host[l];
    return SDETR_OK;
}

extern "C" int sdetr_set_option(const char *name, int value) {
    SDETR_REQUIRE(name, SDETR_ERR_INVALID_ARG, "set_option: null name");
    const auto eq = [&](const char *k) { int i = 0; while (k[i] && k[i] == name[i]) ++i; return k[i] == 0 && name[i] == 0; };
    if (eq("msda_min_blocks")) {
        SDETR_REQUIRE(value >= 2 && value <= 6, SDETR_ERR_INVALID_ARG, "set_option: msda_min_blocks in 2..6");
        g_minb = value;
    } else if (eq("msda_smem_broadcast")) {
        SDETR_REQUIRE(value == 0 || value == 1, SDETR_ERR_INVALID_ARG, "set_option: msda_smem_broadcast in {0,1}");
        g_bcast = value;
    } else if (eq("msda_tma")) {
        SDETR_REQUIRE(value == 0 || value == 1, SDETR_ERR_INVALID_ARG, "set_option: msda_tma in {0,1}");
        g_tma = value;
    } else if (eq("msda_warp_per_item")) {
        SDETR_REQUIRE(value >= 0 && value <= 2, SDETR_ERR_INVALID_ARG, "set_option: msda_warp_per_item in {0,1,2}");
        g_w32 = value;
    } else if (eq("msda_threads")) {
        SDETR_REQUIRE(value == 256 || value == 512 || value == 1024, SDETR_ERR_INVALID_ARG, "set_option: msda_threads in {256,512,1024}");
        g_threads = value;
    } else if (eq("msda_chunk")) {
        SDETR_REQUIRE(value >= 8 && value <= 4096, SDETR_ERR_INVALID_ARG, "set_option: msda_chunk in 8..4096");
        g_chunk = value;
    } else {
        SDETR_REQUIRE(false, SDETR_ERR_INVALID_ARG, "set_option: unknown option %s", name);
    }
    return SDETR_OK;
}

extern "C" int sdetr_msda_forward_ex(const float *value, int64_t value_batch_stride, int64_t value_token_stride,
                                     const int64_t *spatial_shapes, const int64_t *level_start_index,
                                     const float *sampling_loc, const float *attn_weight, float *output, int batch,
                                     int num_value, int num_heads, int head_dim, int num_levels, int num_query,
                                     int num_points, const int32_t *query_order, int schedule,
                                     sdetr_stream_t stream) {
    MsdaFwdParams p{};
    p.value = value, p.v_bstride = value_batch_stride, p.v_tstride = value_token_stride;
    p.shapes = spatial_shapes, p.lsi = level_start_index;
    p.loc = sampling_loc, p.attn = attn_weight, p.out = output, p.order = query_order;
    p.batch = batch, p.nv = num_value, p.heads = num_heads, p.nq = num_query;
    return msda_forward_dispatch(p, false, head_dim, num_levels, num_points, schedule, (cudaStream_t)stream);
}

extern "C" int sdetr_msda_forward(const float *value, const int64_t *spatial_shapes,
                                  const int64_t *level_start_index, const float *sampling_loc,
                                  const float *attn_weight, float *output, int batch, int num_value,
                                  int num_heads, int head_dim, int num_levels, int num_query, int num_points,
                                  sdetr_stream_t stream) {
    return sdetr_msda_forward_ex(value, (int64_t)num_value * num_heads * head_dim, (int64_t)num_heads * head_dim,
                                 spatial_shapes, level_start_index, sampling_loc, attn_weight, output, batch,
                                 num_value, num_heads, head_dim, num_levels, num_query, num_points, nullptr, 0,
                                 stream);
}

static int msda_fused_impl(const float *value, int64_t value_batch_stride, int64_t value_token_stride,
                           const int64_t *spatial_shapes, const int64_t *level_start_index, const float *ref_points, int ref_dim,
                           const float *proj, int64_t proj_stride, float *output, float *loc_out, float *attn_out, int batch,
                           int num_value, int num_heads, int head_dim, int num_levels, int num_query, int num_points,
                           const int32_t *query_order, int schedule, sdetr_stream_t stream) {
    MsdaFwdParams p{};
    p.ref_dim = ref_dim;
    SDETR_REQUIRE(ref_dim == 2 || (ref_dim == 4 && aligned16(ref_points)), SDETR_ERR_INVALID_ARG,
                  "msda_fused_forward: reference points must be (..,2) or 16-byte aligned (..,4) boxes");
    p.value = value, p.v_bstride = value_batch_stride, p.v_tstride = value_token_stride;
    p.shapes = spatial_shapes, p.lsi = level_start_index;
    p.ref = ref_points, p.proj = proj, p.proj_stride = proj_stride, p.loc_out = loc_out, p.attn_out = attn_out;
    p.out = output, p.order = query_order;
    p.batch = batch, p.nv = num_value, p.heads = num_heads, p.nq = num_query;
    SDETR_REQUIRE(proj_stride >= (int64_t)num_heads * num_levels * num_points * 3, SDETR_ERR_INVALID_ARG,
                  "msda_fused_forward: proj_stride too small");
    return msda_forward_dispatch(p, true, head_dim, num_levels, num_points, schedule, (cudaStream_t)stream);
}

extern "C" int sdetr_msda_fused_forward(const float *value, int64_t value_batch_stride, int64_t value_token_stride,
                                        const int64_t *spatial_shapes, const int64_t *level_start_index,
                                        const float *ref_points, const float *proj, int64_t proj_stride,
                                        float *output, float *loc_out, float *attn_out, int batch, int num_value,
                                        int num_heads, int head_dim, int num_levels, int num_query, int num_points,
                                        const int32_t *query_order, int schedule, sdetr_stream_t stream) {
    return msda_fused_impl(value, value_batch_stride, value_token_stride, spatial_shapes, level_start_index, ref_points, 2, proj,
                           proj_stride, output, loc_out, attn_out, batch, num_value, num_heads, head_dim, num_levels, num_query,
                           num_points, query_order, schedule, stream);
}

extern "C" int sdetr_msda_fused_forward_boxes(const float *value, int64_t value_batch_stride, int64_t value_token_stride,
                                              const int64_t *spatial_shapes, const int64_t *level_start_index,
                                              const float *ref_boxes, const float *proj, int64_t proj_stride,
                                              float *output, float *loc_out, float *attn_out, int batch, int num_value,
                                              int num_heads, int head_dim, int num_levels, int num_query, int num_points,
                                              const int32_t *query_order, int schedule, sdetr_stream_t stream) {
    return msda_fused_impl(value, value_batch_stride, value_token_stride, spatial_shapes, level_start_index, ref_boxes, 4, proj,
                           proj_stride, output, loc_out, attn_out, batch, num_value, num_heads, head_dim, num_levels, num_query,
                           num_points, query_order, schedule, stream);
}
