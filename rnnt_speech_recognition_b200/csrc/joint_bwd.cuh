// joint_bwd.cuh -- the two backward contractions of the joint (SURVEY 8 a19: TF autograd through model.py:162-166,
// triggered at run_rnnt.py:284) as hand-written Hopper warpgroup-MMA kernels.  They consume what the forward KEPT: the bf16
// softmax numerators E[row, v] = 2^(y_v - ref_row) (one reference per lattice row) -- the logit gradient of a row is
//     dl[row, :] = rs_row * E'[row, :],     rs_row = g_b * 2^(ref_row + (alpha + beta - ll - lse) * log2 e)
// where E' is E with the row's two special columns (blank, label) replaced by (final value) / rs_row (row_scale_kernel,
// two 2-byte writes per row).  A scale per ROW commutes with both GEMMs, so neither needs a per-element prologue:
//
//   bwd_dz_kernel   dZ[rows,H] = rs_row * (E'[rows,V] . W^T): both operands straight from TMA (K-major), then the row
//                   scale, (1 - tanh^2(enc+pred)) (enc / pred rows staged in shared memory by TMA) and the tile's sums
//                   over u (-> d_enc, accumulated in shared memory along
//                   a run of tiles and stored once) and over t (-> one fp32 partial plane of d_pred per t-block).
//                   Neither dl nor dZ ever exists in HBM.  The epilogue also stores the dW GEMM's A operand
//                   zs[row, :] = [bf16(rs_row * z), bf16(rs_row)], from the tanh it evaluates anyway.
//   bwd_dw_kernel   [dW; db][H+1,V] (+)= zs^T . E'  as a split-K GEMM over the lattice rows, both operands MN-major from
//                   TMA; column H of zs is the row scale itself, so row H of the product is db = sum_rows dl.  Partial
//                   tiles go to fp32 planes (deterministic), summed by sum_planes_kernel.
//
// All operands bf16 (E' needs the exponent range: it is relative to a reference that may lie far below the row maximum),
// fp32 accumulation.  Tile geometry: 16 x 8 lattice tiles (TT = 16 time steps, UU = 8 label positions), row r = tl*8 + ul;
// rows of tile `tile` live at row block slot[tile] of the kept arrays.
#pragma once
#include "joint_tc.cuh"

namespace rb {

constexpr int BW_TT = 16, BW_UU = 8;
constexpr int BWD_THREADS = 288;        // dZ: warps 0-3 / 4-7: consumer warpgroups (M = 64 each) | warp 8: TMA
constexpr int DZ_NC = 128;              // h columns per dZ pass (m64n128 accumulators)
constexpr int DZ_GS_LD = DZ_NC + 8;     // row stride (floats) of the staged gradient tile
constexpr int DZ_MAX_STAGES = 4;
constexpr int DZ_IN_ENC = 0, DZ_IN_PRED = 16 * DZ_NC * 4, DZ_IN_BYTES = DZ_IN_PRED + 8 * DZ_NC * 4;   // a pass's enc / pred slice
constexpr int DW_NV = 256;              // vocabulary columns per dW CTA tile
constexpr int DW_STAGES = 4;            // K steps in flight between the TMA lane and the MMA warpgroups (A + B per stage)

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
    __nv_bfloat16* zs;          // (rows of the kept arrays, zs_ld) the dW operand: column h < H rs * z, column H rs
    int zs_ld;
    // ---- dW kernel
    int nVT, nHB, S;            // DW_NV-column v-tiles, 128-row blocks of [H rows of dW, db], K splits
    float* dWp;                 // (S, H, V) partial planes of dW (zeroed by the host, accumulated over utterance chunks)
    float* dbp;                 // (S, V) partial planes of db
};

// ---------------------------------------------------------------------------------------------------------------
// dZ kernel
// ---------------------------------------------------------------------------------------------------------------
// Work order (identical in both roles): runs = (utterance, t-block) assigned round-robin to CTAs; inside a run the tiles
// along u that have a slot (with windows most tiles of a run have none, at its start as well as its end: both roles skip
// them in lock-step, and a run without any stores its d_enc rows as zeros); inside a tile ceil(H / 128) passes of 128 columns (the last pass of an H % 128 == 64 model reads W rows
// past H as TMA zero fill and stores nothing for them).  A stage = the tile's E' block [128 rows x 64 v] + the pass's W
// rows [128 h x 64 v].  Besides the ring, one input slot holds the pass's enc rows [16 t x 128 h] and pred rows
// [8 u x 128 h] (fp32 boxes, rows past the arrays read as 0) for the epilogue: the TMA lane loads it halfway through the
// pass's K blocks, by when the previous pass's epilogue has released it, so the epilogue finds its inputs in shared
// memory instead of waiting on global loads.
__global__ void __launch_bounds__(BWD_THREADS, 1) bwd_dz_kernel(const __grid_constant__ CUtensorMap tmap_e,
                                                                const __grid_constant__ CUtensorMap tmap_w,
                                                                const __grid_constant__ CUtensorMap tmap_enc,
                                                                const __grid_constant__ CUtensorMap tmap_pred,
                                                                const __grid_constant__ CUtensorMap tmap_zs,
                                                                const BwdParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    const int KBV = p.V >> 6, NPASS = (p.H + DZ_NC - 1) / DZ_NC, stages = p.dz_stages;
    float* gs = reinterpret_cast<float*>(smem + (size_t)stages * 32768);      // [128][DZ_GS_LD] staged gradient rows
    float* dacc = gs + 128 * DZ_GS_LD;                                          // [16][H] the run's d_enc rows
    uint8_t* inp = reinterpret_cast<uint8_t*>(dacc + 16 * p.H);                // the pass's enc / pred slice
    uint64_t* full = reinterpret_cast<uint64_t*>(inp + DZ_IN_BYTES);
    uint64_t* empty = full + DZ_MAX_STAGES;
    uint64_t* in_full = empty + DZ_MAX_STAGES;
    uint64_t* in_empty = in_full + 1;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int i = 0; i < DZ_MAX_STAGES; ++i) { ptx::mbar_init(&full[i], 1); ptx::mbar_init(&empty[i], 2); }
        ptx::mbar_init(in_full, 1); ptx::mbar_init(in_empty, 1);
        ptx::fence_barrier_init();
    }
    if (warp == 8 && lane == 0) {
        ptx::prefetch_tmap(&tmap_e); ptx::prefetch_tmap(&tmap_w); ptx::prefetch_tmap(&tmap_enc); ptx::prefetch_tmap(&tmap_pred);
    }
    if (threadIdx.x == 0) ptx::prefetch_tmap(&tmap_zs);
    for (int i = threadIdx.x; i < 16 * p.H; i += BWD_THREADS) dacc[i] = 0.f;
    __syncthreads();
    const int nruns = p.nb * p.nTb;

    if (warp == 8) {
        // ===================== TMA: A = kept numerators [128 rows x 64 v], B = W rows [128 h x 64 v] =====================
        if (lane == 0) {
            int st = 0; uint32_t ph = 0, iph = 0;
            for (int run = blockIdx.x; run < nruns; run += gridDim.x) {
                const int bl = run / p.nTb, tb = run - bl * p.nTb, b = p.b0 + bl;
                const int Tn = p.xlen[b], Un = p.ylen[b] + 1;
                if (tb * BW_TT >= Tn) continue;
                const int nub = (Un + BW_UU - 1) / BW_UU;
                for (int ub = 0; ub < nub; ++ub) {
                    const int tile = (bl * p.nTb + tb) * p.nUb + ub;
                    const int sl = p.slot ? p.slot[tile] : tile;
                    if (sl < 0) continue;                                    // no slot: outside the windows (or a broken bound)
                    for (int pass = 0; pass < NPASS; ++pass)
                        for (int kb = 0; kb < KBV; ++kb) {
                            if (kb == KBV / 2) {
                                ptx::mbar_wait(in_empty, iph ^ 1);
                                ptx::mbar_arrive_expect_tx(in_full, (uint32_t)DZ_IN_BYTES);
                                ptx::tma_load_2d(inp + DZ_IN_ENC, &tmap_enc, in_full, pass * DZ_NC, b * p.maxT + tb * BW_TT);
                                ptx::tma_load_2d(inp + DZ_IN_PRED, &tmap_pred, in_full, pass * DZ_NC, b * p.maxU + ub * BW_UU);
                                iph ^= 1;
                            }
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
    const uint32_t s_a = ptx::smem_u32(smem), in_a = ptx::smem_u32(inp);
    int st = 0; uint32_t ph = 0, iph = 0;
    for (int run = blockIdx.x; run < nruns; run += gridDim.x) {
        const int bl = run / p.nTb, tb = run - bl * p.nTb, b = p.b0 + bl;
        const int Tn = p.xlen[b], Un = p.ylen[b] + 1;
        if (tb * BW_TT >= Tn) continue;
        const int nub = (Un + BW_UU - 1) / BW_UU;
        for (int ub = 0; ub < nub; ++ub) {
            const int tile = (bl * p.nTb + tb) * p.nUb + ub;
            const int tslot = p.slot ? p.slot[tile] : tile;
            if (tslot < 0) continue;            // as the TMA role: its d_pred partial plane is not written, and not summed
            float rs[2];
#pragma unroll
            for (int ri = 0; ri < 2; ++ri) {    // 0 outside the lattice and the windows
                rs[ri] = __ldg(p.rowscale + (size_t)tslot * 128 + Ra + 8 * ri);
                if (q == 0) p.zs[((size_t)tslot * 128 + Ra + 8 * ri) * p.zs_ld + p.H] = __float2bfloat16_rn(rs[ri]);   // db row
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
                // ---- g = rs * acc * (1 - tanh^2(enc + pred)) -> staged tile, and the dW operand bf16(rs * z) -> zp (0 where
                //      rs == 0, as g: padding outside the lattice never reaches dW).  The previous pass's operand store must
                //      have read the staged tile first.
                if (threadIdx.x == 0) ptx::bulk_wait_group_read<0>();
                ptx::named_bar_sync(1, 256);
                ptx::mbar_wait(in_full, iph);
                iph ^= 1;
                uint32_t zp[2][16];
#pragma unroll
                for (int ri = 0; ri < 2; ++ri) {
                    const int r = Ra + 8 * ri;
                    float* grow = gs + r * DZ_GS_LD + 2 * q;
                    const uint32_t erow = in_a + DZ_IN_ENC + (uint32_t)((r >> 3) * DZ_NC + 2 * q) * 4u,
                                   prow = in_a + DZ_IN_PRED + (uint32_t)((r & 7) * DZ_NC + 2 * q) * 4u;
#pragma unroll
                    for (int j = 0; j < 16; ++j) {
                        const int h = n0 + 8 * j + 2 * q;
                        float2 g = make_float2(0.f, 0.f);
                        zp[ri][j] = 0u;
                        if (rs[ri] != 0.f && h < p.H) {
                            const float2 e = ptx::lds64f(erow + 32u * j), pq = ptx::lds64f(prow + 32u * j);
                            const float z0 = ptx::tanh_approx(e.x + pq.x), z1 = ptx::tanh_approx(e.y + pq.y);
                            const float d0 = acc[4 * j + 2 * ri] * rs[ri], d1 = acc[4 * j + 2 * ri + 1] * rs[ri];
                            g = make_float2(fmaf(-d0 * z0, z0, d0), fmaf(-d1 * z1, z1, d1));
                            zp[ri][j] = ptx::pack_bf16x2(z0 * rs[ri], z1 * rs[ri]);
                        }
                        *reinterpret_cast<float2*>(grow + 8 * j) = g;
                    }
                }
                ptx::named_bar_sync(1, 256);
                if (threadIdx.x == 0) ptx::mbar_arrive(in_empty);      // the input slot has been read
                // ---- sums over u (into the run's d_enc rows) and over t (this t-block's d_pred plane), fixed order, four
                //      columns per thread
                for (int i = threadIdx.x; i < 16 * DZ_NC / 4; i += 256) {
                    const int tl = i / (DZ_NC / 4), col = 4 * (i - tl * (DZ_NC / 4));
                    if (n0 + col >= p.H) continue;
                    float4 sum = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                    for (int ul = 0; ul < BW_UU; ++ul) {
                        const float4 v = *reinterpret_cast<const float4*>(gs + (tl * 8 + ul) * DZ_GS_LD + col);
                        sum.x += v.x; sum.y += v.y; sum.z += v.z; sum.w += v.w;
                    }
                    float4* d = reinterpret_cast<float4*>(dacc + tl * p.H + n0 + col);
                    const float4 a = *d;
                    *d = make_float4(a.x + sum.x, a.y + sum.y, a.z + sum.z, a.w + sum.w);
                }
                for (int i = threadIdx.x; i < BW_UU * DZ_NC / 4; i += 256) {
                    const int ul = i / (DZ_NC / 4), col = 4 * (i - ul * (DZ_NC / 4)), u = ub * BW_UU + ul;
                    if (n0 + col >= p.H || u >= p.maxU) continue;
                    float4 sum = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                    for (int tl = 0; tl < BW_TT; ++tl) {
                        const float4 v = *reinterpret_cast<const float4*>(gs + (tl * 8 + ul) * DZ_GS_LD + col);
                        sum.x += v.x; sum.y += v.y; sum.z += v.z; sum.w += v.w;
                    }
                    *reinterpret_cast<float4*>(p.ppred + (((size_t)tb * p.nb + bl) * p.maxU + u) * p.H + n0 + col) = sum;
                }
                ptx::named_bar_sync(1, 256);
                // ---- the pass's columns of the dW operand: two [128 rows x 64 h] SWIZZLE_128B boxes in the free staged tile,
                //      stored by TMA (columns past H are clipped by the tensor map)
                const uint32_t zs_a = ptx::smem_u32(gs);
#pragma unroll
                for (int ri = 0; ri < 2; ++ri) {
                    const int r = Ra + 8 * ri;
#pragma unroll
                    for (int j = 0; j < 16; ++j)
                        ptx::sts32(zs_a + (uint32_t)((j >> 3) * 16384 + r * 128 + (((j & 7) ^ (r & 7)) << 4) + 4 * q), zp[ri][j]);
                }
                ptx::fence_proxy_async_smem();
                ptx::named_bar_sync(1, 256);
                if (threadIdx.x == 0) {
                    const uint64_t pol = ptx::l2_policy_evict_first();
                    ptx::tma_store_2d(&tmap_zs, gs, n0, tslot * 128, pol);
                    if (n0 + 64 < p.H) ptx::tma_store_2d(&tmap_zs, reinterpret_cast<uint8_t*>(gs) + 16384, n0 + 64, tslot * 128, pol);
                    ptx::bulk_commit_group();
                }
            }
        }
        // ---- the run is complete: its d_enc rows leave once (each entry is read and cleared by the thread that stores it)
        for (int i = threadIdx.x; i < 16 * p.H; i += 256) {
            const int tl = i / p.H, h = i - tl * p.H, t = tb * BW_TT + tl;
            if (t < p.maxT) p.d_enc[((size_t)b * p.maxT + t) * p.H + h] = dacc[i];
            dacc[i] = 0.f;
        }
    }
    if (threadIdx.x == 0) ptx::bulk_wait_group<0>();      // the dW operand has reached global memory
}

struct DzGeom { int stages; size_t smem_bytes; bool ok; };
inline DzGeom dz_geometry(int H) {
    DzGeom g{};
    const size_t fixed = 1024 + (size_t)128 * DZ_GS_LD * 4 + (size_t)16 * H * 4 + DZ_IN_BYTES + (2 * DZ_MAX_STAGES + 2) * 8;
    g.stages = fixed < TC_SMEM_OPTIN ? (int)((TC_SMEM_OPTIN - fixed) / 32768) : 0;
    if (g.stages > DZ_MAX_STAGES) g.stages = DZ_MAX_STAGES;
    g.smem_bytes = fixed + (size_t)g.stages * 32768;
    g.ok = g.stages >= 2;
    return g;
}

// d_pred[b,u,:] = sum over the t-blocks that intersect the utterance of its partial planes (0 for u >= U_b), in t-block
// order.  bwd_dz_kernel writes a plane's rows only for tiles that have a slot, so the others are left out of the sum.
__global__ void __launch_bounds__(256) sum_pred_planes_kernel(const float4* __restrict__ ppred, const int* __restrict__ slot,
                                                              int nTb, int nUb, const int* __restrict__ xlen,
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
                if (slot[(bl * nTb + k) * nUb + u / BW_UU] < 0) continue;
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
// (64 lattice rows: 8 time steps x 8 label positions).  Both operands come from the workspace by TMA:
//   A = the dW operand zs (written by bwd_dz_kernel), rows [64 k] x columns [128 h] as two [64 k x 64 h] SWIZZLE_128B boxes,
//       i.e. MN-major A (one box per consumer warpgroup); columns past H read as zeros, column H is the row scale (db)
//   B = E' [64 k x DW_NV v] as DW_NV / 64 boxes [64 k x 64 v], MN-major.
//   warps 0-7    two consumer warpgroups (64 rows of the block each): wait for a stage, 4 x wgmma m64n256k16, release it
//   warp 8       TMA
// A warpgroup whose 64 rows all lie past row H (the second half of the db-only block when H % 128 == 0) does nothing, and
// its A box is not loaded.  A last v-tile narrower than DW_NV leaves its missing B boxes as zeros: their columns are
// computed as zeros and not stored.
// Each dW / db element is the same chain of k16 products over the same lattice rows, in the same order and on the same
// operand values, whatever DW_NV is: the split plan below is that of 128-column v-tiles (dw_geometry).
constexpr int DW_THREADS = 288;
constexpr int DW_NB = DW_NV / 64;                           // B boxes per stage
constexpr int DW_STAGE_BYTES = 16384 + DW_NB * 8192;        // A [64 k x 128 h] + B [64 k x DW_NV v]
struct DwWork { int vt, hb, split; };
// split-major: the CTAs resident at once cover every (v-tile, h-block) pair of a few splits, so each zs and E' row block
// is fetched from HBM about once and read by the others from L2
__device__ __forceinline__ DwWork dw_decode(const BwdParams& p, int cta) {
    DwWork w;
    w.hb = cta % p.nHB;
    const int rem = cta / p.nHB;
    w.vt = rem % p.nVT;
    w.split = rem / p.nVT;
    return w;
}

__global__ void __launch_bounds__(DW_THREADS, 1) bwd_dw_kernel(const __grid_constant__ CUtensorMap tmap_e,
                                                               const __grid_constant__ CUtensorMap tmap_zs, const BwdParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    // stage st at smem + st * DW_STAGE_BYTES: A boxes (h 0-63 | h 64-127 of the block) at +0 / +8192, B box j at 16384 + j * 8192
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + DW_STAGES * DW_STAGE_BYTES);
    uint64_t* empty = full + DW_STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const DwWork wk = dw_decode(p, blockIdx.x);
    const int v0 = wk.vt * DW_NV, nbox = min(DW_NV, p.V - v0) >> 6, h0 = wk.hb * 128;
    const int nwg = h0 + 64 > p.H ? 1 : 2;                             // consumer warpgroups with a row <= H
    if (threadIdx.x == 0) {
        for (int i = 0; i < DW_STAGES; ++i) { ptx::mbar_init(&full[i], 1); ptx::mbar_init(&empty[i], nwg); }
        ptx::fence_barrier_init();
    }
    if (nbox < DW_NB)   // a narrower last v-tile: the B boxes past it are never loaded and read as zeros
        for (int i = threadIdx.x; i < DW_STAGES * (DW_NB - nbox) * 512; i += DW_THREADS) {
            const int per = (DW_NB - nbox) * 512, st = i / per, k = i - st * per;
            reinterpret_cast<uint4*>(smem + (size_t)st * DW_STAGE_BYTES + 16384 + nbox * 8192)[k] = make_uint4(0u, 0u, 0u, 0u);
        }
    ptx::fence_proxy_async_smem();
    if (warp == 8 && lane == 0) { ptx::prefetch_tmap(&tmap_e); ptx::prefetch_tmap(&tmap_zs); }
    __syncthreads();
    const long long cnt = *p.count;
    const int s_beg = (int)(cnt * wk.split / p.S), s_end = (int)(cnt * (wk.split + 1) / p.S);

    if (warp == 8) {
        // ===================== TMA: per K step the zs boxes and the E' boxes =====================
        if (lane == 0) {
            int st = 0; uint32_t ph = 0;
            for (int step = 2 * s_beg; step < 2 * s_end; ++step) {
                ptx::mbar_wait(&empty[st], ph ^ 1);
                ptx::mbar_arrive_expect_tx(&full[st], (uint32_t)(nwg + nbox) * 8192u);
                uint8_t* sb = smem + (size_t)st * DW_STAGE_BYTES;
                for (int w = 0; w < nwg; ++w) ptx::tma_load_2d(sb + w * 8192, &tmap_zs, &full[st], h0 + 64 * w, step * 64);
                for (int j = 0; j < nbox; ++j) ptx::tma_load_2d(sb + 16384 + j * 8192, &tmap_e, &full[st], v0 + 64 * j, step * 64);
                if (++st == DW_STAGES) { st = 0; ph ^= 1; }
            }
        }
        return;
    }

    // ===================== consumer warpgroups: D[64 h x DW_NV v] += A[64 h x 64 k] . E'[64 k x DW_NV v] =====================
    const int wg = warp >> 2, t128 = threadIdx.x & 127, q = lane & 3;
    if (h0 + wg * 64 > p.H) return;
    const uint32_t s_a = ptx::smem_u32(smem);
    float acc[DW_NV / 2];
#pragma unroll
    for (int i = 0; i < DW_NV / 2; ++i) acc[i] = 0.f;
    int st = 0, prev = -1; uint32_t ph = 0;
    for (int step = 2 * s_beg; step < 2 * s_end; ++step) {
        ptx::mbar_wait_warp(&full[st], ph);
        const uint32_t sa = s_a + (uint32_t)st * DW_STAGE_BYTES;
        const uint64_t ad = ptx::gmma_desc_mn_sw128(sa + (uint32_t)wg * 8192u, 8192u), bd = ptx::gmma_desc_mn_sw128(sa + 16384u, 8192u);
        ptx::wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k)   // K = 16 lattice rows per MMA: 16 x 128 B of A and of every B box
            ptx::wgmma_m64n256_bf16<1, 1>(acc, ad + (uint64_t)(k * 128), bd + (uint64_t)(k * 128), 1u);
        ptx::wgmma_commit();
        ptx::wgmma_wait<1>();        // the previous step's MMAs have retired: its stage is free
        if (prev >= 0 && t128 == 0) ptx::mbar_arrive(&empty[prev]);
        prev = st;
        if (++st == DW_STAGES) { st = 0; ph ^= 1; }
    }
    ptx::wgmma_wait<0>();
    if (prev >= 0 && t128 == 0) ptx::mbar_arrive(&empty[prev]);
    ptx::fence_regs(acc);
    if (s_end <= s_beg) return;
    // ---- epilogue: rows (Ra, Ra + 8) x DW_NV / 4 columns of the block -> accumulated into the split's partial plane
    const int Ra = h0 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
    for (int ri = 0; ri < 2; ++ri) {
        const int hr = Ra + 8 * ri;
        if (hr > p.H) continue;
        float* dst = hr < p.H ? p.dWp + ((size_t)wk.split * p.H + hr) * p.V : p.dbp + (size_t)wk.split * p.V;
#pragma unroll
        for (int j = 0; j < DW_NV / 8; ++j) {
            const int v = v0 + 8 * j + 2 * q;
            if (v >= p.V) continue;
            float2* d2 = reinterpret_cast<float2*>(dst + v);
            const float2 x = *d2;
            *d2 = make_float2(x.x + acc[4 * j + 2 * ri], x.y + acc[4 * j + 2 * ri + 1]);
        }
    }
}

struct DwGeom { int nVT, nHB, S, nCT; size_t smem_bytes; };
// S: lattice-row splits for about four waves of 128-column CTAs.  Besides balancing the grid this bounds the length of
// each fp32 accumulation chain (db[blank] is a same-sign sum over every lattice row: at C3 one split per SM would chain
// 1 M rows).  A pure function of (H, V), as the workspace holds S planes; it stays that of 128-column v-tiles (nVT) so
// that the split boundaries, and with them dW's bits, do not depend on the CTA tile width (nCT v-tiles of DW_NV).
inline DwGeom dw_geometry(int H, int V) {
    DwGeom g{};
    g.nVT = (V + 127) / 128;
    g.nCT = (V + DW_NV - 1) / DW_NV;
    g.nHB = H / 128 + 1;                    // rows 0 .. H (row H: db)
    g.S = 4 * TC_SMS / (g.nVT * g.nHB);
    if (g.S < 1) g.S = 1;
    if (g.S > 64) g.S = 64;
    g.smem_bytes = 1024 + (size_t)DW_STAGES * DW_STAGE_BYTES + 2 * DW_STAGES * 8;
    return g;
}

}  // namespace rb
