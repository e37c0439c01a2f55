// joint_bwd.cuh -- the two backward contractions of the joint (SURVEY 8 a19: TF autograd through model.py:162-166,
// triggered at run_rnnt.py:284) as hand-written Hopper warpgroup-MMA kernels.  They consume what the forward KEPT: the bf16
// softmax numerators E[row, v] = 2^(y_v - ref_row) (one reference per lattice row) -- the logit gradient of a row is
//     dl[row, :] = rs_row * E'[row, :],     rs_row = g_b * 2^(ref_row + (alpha + beta - ll - lse) * log2 e)
// where E' is E with the row's two special columns (blank, label) replaced by (final value) / rs_row (row_scale_kernel,
// two 2-byte writes per row).  A scale per ROW commutes with both GEMMs, so neither needs a per-element prologue:
//
//   bwd_dz_kernel   dZ[rows,H] = rs_row * (E'[rows,V] . W^T): both operands straight from TMA (K-major), then the row
//                   scale, (1 - tanh^2(enc+pred)) and the tile's sums over u (-> d_enc, accumulated in shared memory along
//                   a run of tiles and stored once) and over t (-> one fp32 partial plane of d_pred per t-block).
//                   Neither dl nor dZ ever exists in HBM.
//   bwd_dw_kernel   [dW; db][H+1,V] (+)= ([rs_row * z, rs_row])^T . E'  as a split-K GEMM over the lattice rows: the A operand
//                   is REGENERATED from enc/pred by the consumer warpgroups themselves (tanh, times the row scale, K-major
//                   SWIZZLE_128B) while the previous K step's MMAs run; row H of A is the row scale itself, so row H of the
//                   product is db = sum_rows dl.  The B operand is E' loaded MN-major by TMA.  Partial tiles go to fp32
//                   planes (deterministic), summed by sum_planes_kernel.
//
// All operands bf16 (E' needs the exponent range: it is relative to a reference that may lie far below the row maximum),
// fp32 accumulation.  Tile geometry: 16 x 8 lattice tiles (TT = 16 time steps, UU = 8 label positions), row r = tl*8 + ul;
// rows of tile `tile` live at row block slot[tile] of the kept arrays.
#pragma once
#include "joint_tc.cuh"

namespace rb {

constexpr int BW_TT = 16, BW_UU = 8;
constexpr int BWD_THREADS = 288;        // warps 0-3 / 4-7: consumer warpgroups (M = 64 each) | warp 8: TMA
constexpr int DZ_NC = 128;              // h columns per dZ pass (m64n128 accumulators)
constexpr int DZ_GS_LD = DZ_NC + 8;     // row stride (floats) of the staged gradient tile
constexpr int DZ_MAX_STAGES = 4;
constexpr int DW_NV = 128;              // vocabulary columns per dW output tile
constexpr int DW_STAGES = 4;

struct BwdParams {
    const float* enc; const float* pred;
    const int* xlen; const int* ylen;
    int maxT, maxU, H, V;
    int nTb, nUb, b0, nb;
    const int* slot;            // tile -> row block of the kept arrays (-1: tile outside the valid lattice)
    const int4* slot_meta;      // per compact slot {first enc row, first pred row, #t rows, #u rows} of the tile
    const int* count;           // number of valid tiles (device word)
    const float* rowscale;      // per row of the kept arrays: rs_row (0 for rows outside the lattice)   [row_scale_kernel]
    // ---- dZ kernel
    int dz_stages;
    float* d_enc;               // (B, maxT, H), rows of this launch's utterances are fully written
    float* ppred;               // (nTb, nb, maxU, H) partial planes of d_pred
    // ---- dW kernel
    int nVT, nHB, S;            // v-tiles, 128-row blocks of [H rows of dW, db], K splits
    float* dWp;                 // (S, H, V) partial planes of dW (zeroed by the host, accumulated over utterance chunks)
    float* dbp;                 // (S, V) partial planes of db
};

// ---------------------------------------------------------------------------------------------------------------
// dZ kernel
// ---------------------------------------------------------------------------------------------------------------
// Work order (identical in both roles): runs = (utterance, t-block) assigned round-robin to CTAs; inside a run the valid
// tiles along u; inside a tile ceil(H / 128) passes of 128 columns (the last pass of an H % 128 == 64 model reads W rows
// past H as TMA zero fill and stores nothing for them).  A stage = the tile's E' block [128 rows x 64 v] + the pass's W
// rows [128 h x 64 v].
__global__ void __launch_bounds__(BWD_THREADS, 1) bwd_dz_kernel(const __grid_constant__ CUtensorMap tmap_e,
                                                                const __grid_constant__ CUtensorMap tmap_w,
                                                                const BwdParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    const int KBV = p.V >> 6, NPASS = (p.H + DZ_NC - 1) / DZ_NC, stages = p.dz_stages;
    float* gs = reinterpret_cast<float*>(smem + (size_t)stages * 32768);      // [128][DZ_GS_LD] staged gradient rows
    float* dacc = gs + 128 * DZ_GS_LD;                                          // [16][H] the run's d_enc rows
    uint64_t* full = reinterpret_cast<uint64_t*>(dacc + 16 * p.H);
    uint64_t* empty = full + DZ_MAX_STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int i = 0; i < DZ_MAX_STAGES; ++i) { ptx::mbar_init(&full[i], 1); ptx::mbar_init(&empty[i], 2); }
        ptx::fence_barrier_init();
    }
    if (warp == 8 && lane == 0) { ptx::prefetch_tmap(&tmap_e); ptx::prefetch_tmap(&tmap_w); }
    for (int i = threadIdx.x; i < 16 * p.H; i += BWD_THREADS) dacc[i] = 0.f;
    __syncthreads();
    const int nruns = p.nb * p.nTb;

    if (warp == 8) {
        // ===================== TMA: A = kept numerators [128 rows x 64 v], B = W rows [128 h x 64 v] =====================
        if (lane == 0) {
            int st = 0; uint32_t ph = 0;
            for (int run = blockIdx.x; run < nruns; run += gridDim.x) {
                const int bl = run / p.nTb, tb = run - bl * p.nTb, b = p.b0 + bl;
                const int Tn = p.xlen[b], Un = p.ylen[b] + 1;
                if (tb * BW_TT >= Tn) continue;
                const int nub = (Un + BW_UU - 1) / BW_UU;
                for (int ub = 0; ub < nub; ++ub) {
                    const int tile = (bl * p.nTb + tb) * p.nUb + ub;
                    const int sl = max(p.slot ? p.slot[tile] : tile, 0);   // a slot-less tile (broken bound) has rs = 0 everywhere
                    for (int pass = 0; pass < NPASS; ++pass)
                        for (int kb = 0; kb < KBV; ++kb) {
                            ptx::mbar_wait(&empty[st], ph ^ 1);
                            ptx::mbar_arrive_expect_tx(&full[st], 32768u);
                            uint8_t* sa = smem + (size_t)st * 32768;
                            ptx::tma_load_2d(sa, &tmap_e, &full[st], kb * 64, sl * 128);
                            ptx::tma_load_2d(sa + 16384, &tmap_w, &full[st], kb * 64, pass * DZ_NC);
                            if (++st == stages) { st = 0; ph ^= 1; }
                        }
                }
            }
        }
        return;
    }

    // ===================== consumer warpgroups: D[64 x 128] += A[64 x 64] . B[128 x 64]^T, then the epilogue =====================
    const int wg = threadIdx.x >> 7, t128 = threadIdx.x & 127, q = lane & 3;
    const int Ra = wg * 64 + (warp & 3) * 16 + (lane >> 2);          // rows Ra and Ra + 8 of the tile
    const uint32_t s_a = ptx::smem_u32(smem);
    int st = 0; uint32_t ph = 0;
    for (int run = blockIdx.x; run < nruns; run += gridDim.x) {
        const int bl = run / p.nTb, tb = run - bl * p.nTb, b = p.b0 + bl;
        const int Tn = p.xlen[b], Un = p.ylen[b] + 1;
        if (tb * BW_TT >= Tn) continue;
        const int nub = (Un + BW_UU - 1) / BW_UU;
        for (int ub = 0; ub < nub; ++ub) {
            const int tile = (bl * p.nTb + tb) * p.nUb + ub;
            const int tslot = p.slot ? p.slot[tile] : tile;               // < 0 only after a broken valid_tile_bound promise
            float rs[2];
            const float* erow[2];
            const float* prow[2];
#pragma unroll
            for (int ri = 0; ri < 2; ++ri) {
                const int r = Ra + 8 * ri, t = tb * BW_TT + (r >> 3), u = ub * BW_UU + (r & 7);
                rs[ri] = tslot >= 0 ? __ldg(p.rowscale + (size_t)tslot * 128 + r) : 0.f;   // 0 outside the lattice
                erow[ri] = p.enc + ((size_t)b * p.maxT + min(t, p.maxT - 1)) * p.H;
                prow[ri] = p.pred + ((size_t)b * p.maxU + min(u, p.maxU - 1)) * p.H;
            }
            for (int pass = 0; pass < NPASS; ++pass) {
                const int n0 = pass * DZ_NC;
                float acc[64];
#pragma unroll
                for (int i = 0; i < 64; ++i) acc[i] = 0.f;
                int prev = -1;
                for (int kb = 0; kb < KBV; ++kb) {
                    ptx::mbar_wait(&full[st], ph);
                    const uint32_t sa = s_a + (uint32_t)st * 32768u;
                    const uint64_t ad = ptx::gmma_desc_k_sw128(sa + (uint32_t)wg * 8192u), bd = ptx::gmma_desc_k_sw128(sa + 16384u);
                    ptx::wgmma_fence();
#pragma unroll
                    for (int k = 0; k < 4; ++k) ptx::wgmma_m64n128_bf16<0>(acc, ad + (uint64_t)(k * 2), bd + (uint64_t)(k * 2), 1u);
                    ptx::wgmma_commit();
                    ptx::wgmma_wait<1>();
                    if (prev >= 0 && t128 == 0) ptx::mbar_arrive(&empty[prev]);
                    prev = st;
                    if (++st == stages) { st = 0; ph ^= 1; }
                }
                ptx::wgmma_wait<0>();
                if (t128 == 0) ptx::mbar_arrive(&empty[prev]);
                ptx::fence_regs(acc);
                // ---- g = rs * acc * (1 - tanh^2(enc + pred)) -> staged tile
#pragma unroll
                for (int ri = 0; ri < 2; ++ri) {
                    float* grow = gs + (Ra + 8 * ri) * DZ_GS_LD + 2 * q;
#pragma unroll
                    for (int j = 0; j < 16; ++j) {
                        const int h = n0 + 8 * j + 2 * q;
                        float2 g = make_float2(0.f, 0.f);
                        if (rs[ri] != 0.f && h < p.H) {
                            const float2 e = __ldg(reinterpret_cast<const float2*>(erow[ri] + h)),
                                         pq = __ldg(reinterpret_cast<const float2*>(prow[ri] + h));
                            const float z0 = ptx::tanh_approx(e.x + pq.x), z1 = ptx::tanh_approx(e.y + pq.y);
                            const float d0 = acc[4 * j + 2 * ri] * rs[ri], d1 = acc[4 * j + 2 * ri + 1] * rs[ri];
                            g = make_float2(fmaf(-d0 * z0, z0, d0), fmaf(-d1 * z1, z1, d1));
                        }
                        *reinterpret_cast<float2*>(grow + 8 * j) = g;
                    }
                }
                ptx::named_bar_sync(1, 256);
                // ---- sums over u (into the run's d_enc rows) and over t (this t-block's d_pred plane), fixed order
                for (int i = threadIdx.x; i < 16 * DZ_NC; i += 256) {
                    const int tl = i / DZ_NC, col = i - tl * DZ_NC;
                    if (n0 + col >= p.H) continue;
                    float sum = 0.f;
#pragma unroll
                    for (int ul = 0; ul < BW_UU; ++ul) sum += gs[(tl * 8 + ul) * DZ_GS_LD + col];
                    dacc[tl * p.H + n0 + col] += sum;
                }
                for (int i = threadIdx.x; i < BW_UU * DZ_NC; i += 256) {
                    const int ul = i / DZ_NC, col = i - ul * DZ_NC, u = ub * BW_UU + ul;
                    if (n0 + col >= p.H || u >= p.maxU) continue;
                    float sum = 0.f;
#pragma unroll
                    for (int tl = 0; tl < BW_TT; ++tl) sum += gs[(tl * 8 + ul) * DZ_GS_LD + col];
                    p.ppred[(((size_t)tb * p.nb + bl) * p.maxU + u) * p.H + n0 + col] = sum;
                }
                ptx::named_bar_sync(1, 256);
            }
        }
        // ---- the run is complete: its d_enc rows leave once (each entry is read and cleared by the thread that stores it)
        for (int i = threadIdx.x; i < 16 * p.H; i += 256) {
            const int tl = i / p.H, h = i - tl * p.H, t = tb * BW_TT + tl;
            if (t < p.maxT) p.d_enc[((size_t)b * p.maxT + t) * p.H + h] = dacc[i];
            dacc[i] = 0.f;
        }
    }
}

struct DzGeom { int stages; size_t smem_bytes; bool ok; };
inline DzGeom dz_geometry(int H) {
    DzGeom g{};
    const size_t fixed = 1024 + (size_t)128 * DZ_GS_LD * 4 + (size_t)16 * H * 4 + 2 * DZ_MAX_STAGES * 8;
    g.stages = fixed < TC_SMEM_OPTIN ? (int)((TC_SMEM_OPTIN - fixed) / 32768) : 0;
    if (g.stages > DZ_MAX_STAGES) g.stages = DZ_MAX_STAGES;
    g.smem_bytes = fixed + (size_t)g.stages * 32768;
    g.ok = g.stages >= 2;
    return g;
}

// d_pred[b,u,:] = sum over the t-blocks that intersect the utterance of its partial planes (0 for u >= U_b)
__global__ void __launch_bounds__(256) sum_pred_planes_kernel(const float4* __restrict__ ppred, const int* __restrict__ xlen,
                                                              const int* __restrict__ ylen, int b0, int nb, int maxU, int H4,
                                                              float4* __restrict__ d_pred) {
    const size_t n4 = (size_t)nb * maxU * H4;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
        const int bl = (int)(i / ((size_t)maxU * H4)), u = (int)((i / H4) % maxU), b = b0 + bl;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        if (u < ylen[b] + 1) {
            const int ntb = (xlen[b] + BW_TT - 1) / BW_TT;
#pragma unroll 4
            for (int k = 0; k < ntb; ++k) {
                const float4 v = ppred[(size_t)k * n4 + i];
                acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
            }
        }
        d_pred[(size_t)b0 * maxU * H4 + i] = acc;
    }
}

// ---------------------------------------------------------------------------------------------------------------
// dW kernel
// ---------------------------------------------------------------------------------------------------------------
// CTA = (v-tile of DW_NV columns, 128-row block of [dW rows 0..H-1, db], split of the lattice rows).  K step = half a tile
// (64 lattice rows: 8 time steps x 8 label positions).  Each consumer warpgroup owns 64 rows of the block and produces
// their A tile [64 h x 64 k] (double-buffered) while the previous step's MMAs run.
struct DwWork { int vt, hb, split; };
__device__ __forceinline__ DwWork dw_decode(const BwdParams& p, int cta) {
    DwWork w;
    const int per_vt = p.nHB * p.S;
    w.vt = cta / per_vt;
    const int rem = cta - w.vt * per_vt;
    w.hb = rem / p.S;
    w.split = rem - w.hb * p.S;
    return w;
}

__global__ void __launch_bounds__(BWD_THREADS, 1) bwd_dw_kernel(const __grid_constant__ CUtensorMap tmap_e, const BwdParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    // B stages: [64 k x 128 v] as two [64 k x 64 v] boxes (MN-major, SW128) | A: [warpgroup][buffer][64 h x 64 k] K-major
    uint8_t* bsm = smem;
    uint8_t* asm_ = smem + DW_STAGES * 16384;
    uint64_t* full = reinterpret_cast<uint64_t*>(asm_ + 4 * 8192);
    uint64_t* empty = full + DW_STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const DwWork wk = dw_decode(p, blockIdx.x);
    const int v0 = wk.vt * DW_NV, nbox = min(DW_NV, p.V - v0) >> 6;
    if (threadIdx.x == 0) {
        for (int i = 0; i < DW_STAGES; ++i) { ptx::mbar_init(&full[i], 1); ptx::mbar_init(&empty[i], 2); }
        ptx::fence_barrier_init();
    }
    if (nbox == 1)      // a 64-wide last v-tile: the second box of every stage is never loaded and reads as zeros
        for (int i = threadIdx.x; i < DW_STAGES * 512; i += BWD_THREADS)
            reinterpret_cast<uint4*>(bsm + (size_t)(i >> 9) * 16384 + 8192)[i & 511] = make_uint4(0u, 0u, 0u, 0u);
    ptx::fence_proxy_async_smem();
    if (warp == 8 && lane == 0) ptx::prefetch_tmap(&tmap_e);
    __syncthreads();
    const long long cnt = *p.count;
    const int s_beg = (int)(cnt * wk.split / p.S), s_end = (int)(cnt * (wk.split + 1) / p.S);

    if (warp == 8) {
        // ===================== TMA: B = kept numerators, boxes [64 rows x 64 v] (rows = K) =====================
        if (lane == 0) {
            int st = 0; uint32_t ph = 0;
            for (int s = s_beg; s < s_end; ++s)
                for (int half = 0; half < 2; ++half) {
                    ptx::mbar_wait(&empty[st], ph ^ 1);
                    ptx::mbar_arrive_expect_tx(&full[st], (uint32_t)nbox * 8192u);
                    for (int j = 0; j < nbox; ++j)
                        ptx::tma_load_2d(bsm + (size_t)st * 16384 + j * 8192, &tmap_e, &full[st], v0 + 64 * j, s * 128 + half * 64);
                    if (++st == DW_STAGES) { st = 0; ph ^= 1; }
                }
        }
        return;
    }

    // ===================== consumer warpgroups: produce A, D[64 h x 128 v] += A[64 h x 64 k] . E'[64 k x 128 v] =====================
    const int wg = threadIdx.x >> 7, t128 = threadIdx.x & 127, q = lane & 3;
    const int hl = t128 & 63, hq = t128 >> 6;                         // A row of this thread; which 4 of a K step's 8 time rows
    const int h = wk.hb * 128 + wg * 64 + hl;
    const int kind = h < p.H ? 0 : (h == p.H ? 1 : 2);                // z row | row-scale row (db) | zero row
    const int hc = min(h, p.H - 1);
    const uint32_t a_a = ptx::smem_u32(asm_) + (uint32_t)wg * 16384u, b_a = ptx::smem_u32(bsm);
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    int st = 0, prev = -1; uint32_t ph = 0, it = 0;
    for (int s = s_beg; s < s_end; ++s) {
        // this slot's inputs: 8 pred rows and 8 enc rows (4 per half) of column h; rows past the padded arrays are clamped
        // (their row scale is 0)
        const int4 m = __ldg(p.slot_meta + s);
        float pv[8], ev[8];
        if (kind == 0) {
#pragma unroll
            for (int k = 0; k < 8; ++k) pv[k] = __ldg(p.pred + (size_t)(m.y + min(k, m.w - 1)) * p.H + hc);
#pragma unroll
            for (int k = 0; k < 8; ++k) ev[k] = __ldg(p.enc + (size_t)(m.x + min((k >> 2) * 8 + hq * 4 + (k & 3), m.z - 1)) * p.H + hc);
        }
        for (int half = 0; half < 2; ++half, ++it) {
            const uint32_t abuf = a_a + (it & 1) * 8192u;
            const float* rsp = p.rowscale + (size_t)s * 128 + half * 64;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int tl = hq * 4 + j;
                const float4 r0 = __ldg(reinterpret_cast<const float4*>(rsp + tl * 8)), r1 = __ldg(reinterpret_cast<const float4*>(rsp + tl * 8 + 4));
                const float rsv[8] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w};
                float z[8];
#pragma unroll
                for (int k = 0; k < 8; ++k)
                    z[k] = kind == 0 ? ptx::tanh_approx(ev[half * 4 + j] + pv[k]) * rsv[k] : (kind == 1 ? rsv[k] : 0.f);
                ptx::sts128(abuf + (uint32_t)(hl * 128 + ((tl ^ (hl & 7)) << 4)),
                            make_uint4(ptx::pack_bf16x2(z[0], z[1]), ptx::pack_bf16x2(z[2], z[3]), ptx::pack_bf16x2(z[4], z[5]),
                                       ptx::pack_bf16x2(z[6], z[7])));
            }
            ptx::fence_proxy_async_smem();
            ptx::named_bar_sync(1 + wg, 128);
            ptx::mbar_wait(&full[st], ph);
            const uint64_t ad = ptx::gmma_desc_k_sw128(abuf), bd = ptx::gmma_desc_mn_sw128(b_a + (uint32_t)st * 16384u, 8192u);
            ptx::wgmma_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k)   // K = 16 lattice rows per MMA: 32 B along A's rows, 16 x 128 B of B
                ptx::wgmma_m64n128_bf16<1>(acc, ad + (uint64_t)(k * 2), bd + (uint64_t)(k * 128), 1u);
            ptx::wgmma_commit();
            ptx::wgmma_wait<1>();        // the previous step's MMAs have retired: its B stage and A buffer are free
            if (prev >= 0 && t128 == 0) ptx::mbar_arrive(&empty[prev]);
            prev = st;
            if (++st == DW_STAGES) { st = 0; ph ^= 1; }
        }
    }
    ptx::wgmma_wait<0>();
    if (prev >= 0 && t128 == 0) ptx::mbar_arrive(&empty[prev]);
    ptx::fence_regs(acc);
    if (s_end <= s_beg) return;
    // ---- epilogue: rows (Ra, Ra + 8) x 32 columns of the block -> accumulated into the split's partial plane
    const int Ra = wk.hb * 128 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
    for (int ri = 0; ri < 2; ++ri) {
        const int hr = Ra + 8 * ri;
        if (hr > p.H) continue;
        float* dst = hr < p.H ? p.dWp + ((size_t)wk.split * p.H + hr) * p.V : p.dbp + (size_t)wk.split * p.V;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            const int v = v0 + 8 * j + 2 * q;
            if (v >= p.V) continue;
            float2* d2 = reinterpret_cast<float2*>(dst + v);
            const float2 x = *d2;
            *d2 = make_float2(x.x + acc[4 * j + 2 * ri], x.y + acc[4 * j + 2 * ri + 1]);
        }
    }
}

struct DwGeom { int nVT, nHB, S; size_t smem_bytes; };
// S: lattice-row splits for about four waves of CTAs.  Besides balancing the grid this bounds the length of each fp32
// accumulation chain (db[blank] is a same-sign sum over every lattice row: at C3 one split per SM would chain 1 M rows).
// A pure function of (H, V), as the workspace holds S planes.
inline DwGeom dw_geometry(int H, int V) {
    DwGeom g{};
    g.nVT = (V + DW_NV - 1) / DW_NV;
    g.nHB = H / 128 + 1;                    // rows 0 .. H (row H: db)
    g.S = 4 * TC_SMS / (g.nVT * g.nHB);
    if (g.S < 1) g.S = 1;
    if (g.S > 64) g.S = 64;
    g.smem_bytes = 1024 + (size_t)DW_STAGES * 16384 + 4 * 8192 + 2 * DW_STAGES * 8;
    return g;
}

}  // namespace rb
