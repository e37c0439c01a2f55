// joint_fwd.cuh -- the fused joint FORWARD kernel (SURVEY 8 a1-a5, a11: model.py:158-166 + the log-softmax and gather of
// gpu_rnnt.h:73-80 / gpu_rnnt_kernel.h:5-9) on Hopper warpgroup MMA.
//
// One persistent CTA per SM loops over 128-cell lattice tiles (16 time steps x 8 label positions).  Per tile the two
// consumer warpgroups each build their 64 rows of the A operand z = tanh(enc + pred) as fp16 in shared memory (K-major,
// SWIZZLE_128B, all H columns: at most 192 KB at H = 768), then walk the vocabulary in 64-column chunks: wgmma
// m64n64k16 against W^T (fp16) K blocks that one TMA warp streams through a ring, accumulators in registers, and the
// chunk's softmax statistics in the epilogue.  The (B,T,U,H) activations and the (B,T,U,V) logits never exist in HBM.
//
// Operand format: fp16 (z in [-1, 1], W ~ 1/sqrt(H): both far inside the fp16 range; 11-bit significand).  tanh is
// tanh.approx.f32 (2^-11 relative).
//
// Warps 0-3 / 4-7: consumer warpgroups (tile rows 0-63 / 64-127) | warp 8: W^T TMA.
//
// MODE 0  forward: lse + (blank, label) log-probs per cell; nothing else leaves the SM
// MODE 2  forward that KEEPS its activations (rnntb200JointDesc.keep_activations, and the backward's per-chunk
//         recompute): MODE 0 + the softmax numerators E[row, v] = 2^(y_v - ref_row) as bf16, all columns of a row against
//         ONE reference ref_row, and ref_row itself.  ref_row starts as the maximum of the row's first 32 logits; a chunk
//         holding a logit more than 2^FWD_REBASE above it raises it by whole octaves to at least that chunk's maximum
//         (rescaling the numerators already stored), so every stored numerator is at most 2^FWD_REBASE and the row
//         maximum is at most ref_row + FWD_REBASE.  bf16 keeps its 8 significant bits over the whole exponent range, so
//         any reference in that window works.  The logit gradients are then row_scale * E: the two backward GEMMs take E
//         straight from TMA.
//         Both modes form the softmax sum and the reference with the same arithmetic, so they give identical costs.
#pragma once
#include <cuda_fp16.h>
#include "joint_tc.cuh"

namespace rb {

constexpr int FWD_THREADS = 288;
constexpr int FWD_NC = 64;              // vocabulary columns per chunk (one m64n64 accumulator per warpgroup)
constexpr int FWD_MAX_STAGES = 8;
constexpr float FWD_REBASE = 64.f;      // log2 units: largest stored numerator 2^64, row maximum <= ref_row + 64

struct FwdGeom { int stages; size_t smem_bytes; bool ok; };
inline FwdGeom fwd_geometry(int H, int V) {
    FwdGeom g{};
    if (H % 64 || V % 64 || H < 64 || H > 64 * TC_MAX_KB) return g;
    const size_t z_bytes = (size_t)(H / 64) * 16384;
    const size_t fixed = 1024 + z_bytes + 256;
    if (fixed + 2 * 8192 > TC_SMEM_OPTIN) return g;
    g.stages = (int)((TC_SMEM_OPTIN - fixed) / 8192);
    if (g.stages > FWD_MAX_STAGES) g.stages = FWD_MAX_STAGES;
    g.smem_bytes = fixed + (size_t)g.stages * 8192;
    g.ok = g.stages >= 2;
    return g;
}

// Rebase of one row's reference (MODE comment above), called by all 32 lanes of the warp when a chunk holds a logit more
// than 2^FWD_REBASE above the reference of any of its rows.  The quad takes a new reference a whole number of octaves
// above the old one, at least the chunk's row maximum, and (MODE 2) each lane scales the numerators it stored for the
// row's earlier chunks by that power of two: it reads back its own stores.  Inlined behind a warp-uniform branch:
// as a real call (__noinline__) the keeping forward took 0.3 ms (4 %) longer at BASELINE C3, on an H100 80GB HBM3 at
// 700 W, although ordinary inputs never take the branch.
template <int MODE>
__device__ __forceinline__ float fwd_rebase(float gm, float ref, __nv_bfloat16* dl, long long row, int V, int q, int c) {
    float qm = fmaxf(gm, __shfl_xor_sync(0xffffffffu, gm, 1));
    qm = fmaxf(qm, __shfl_xor_sync(0xffffffffu, qm, 2));
    if (!(qm - ref > FWD_REBASE)) return ref;
    const float sh = ceilf(qm - ref);
    if (MODE == 2 && row >= 0) {
        const float f = ldexpf(1.f, -(int)fminf(sh, 200.f));
        uint32_t* w = reinterpret_cast<uint32_t*>(dl + row * V + 2 * q);
        for (int cc = 0; cc < c; ++cc)
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const uint32_t v = w[cc * (FWD_NC / 2) + 4 * j];
                w[cc * (FWD_NC / 2) + 4 * j] = ptx::pack_bf16x2(__uint_as_float(v << 16) * f, __uint_as_float(v & 0xffff0000u) * f);
            }
    }
    return ref + sh;
}

template <int MODE>
__global__ void __launch_bounds__(FWD_THREADS, 1) joint_fwd_kernel(const __grid_constant__ CUtensorMap tmap_wt,
                                                                   const JointTcParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    const int KB = p.KB, NCH = p.V / FWD_NC, stages = p.stages;
    uint8_t* zsm = smem;                                            // KB x [128 rows x 64 k] fp16, SW128 K-major
    uint8_t* wsm = zsm + (size_t)KB * 16384;                        // stages x [64 v x 64 k] fp16, SW128 K-major (TMA)
    uint64_t* full = reinterpret_cast<uint64_t*>(wsm + (size_t)stages * 8192);
    uint64_t* empty = full + FWD_MAX_STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int i = 0; i < FWD_MAX_STAGES; ++i) { ptx::mbar_init(&full[i], 1); ptx::mbar_init(&empty[i], 2); }
        ptx::fence_barrier_init();
    }
    if (warp == 8 && lane == 0) ptx::prefetch_tmap(&tmap_wt);
    __syncthreads();
    const int ntiles = p.nb * p.nTb * p.nUb;

    if (warp == 8) {
        // ===================== W^T TMA: per valid tile, every (chunk, K block) box in the consumers' order =====================
        if (lane == 0) {
            int st = 0; uint32_t ph = 0;
            for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
                if (!decode_tile(p, tile).valid) continue;
                for (int c = 0; c < NCH; ++c)
                    for (int kb = 0; kb < KB; ++kb) {
                        ptx::mbar_wait(&empty[st], ph ^ 1);
                        ptx::mbar_arrive_expect_tx(&full[st], 8192u);
                        ptx::tma_load_2d(wsm + (size_t)st * 8192, &tmap_wt, &full[st], kb * 64, c * FWD_NC);
                        if (++st == stages) { st = 0; ph ^= 1; }
                    }
            }
        }
        return;
    }

    // ===================== consumer warpgroups =====================
    constexpr float LOG2E = 1.4426950408889634f, LN2 = 0.6931471805599453f;
    const int wg = threadIdx.x >> 7, t128 = threadIdx.x & 127, q = lane & 3;
    const int Ra = wg * 64 + (warp & 3) * 16 + (lane >> 2);          // this thread's two tile rows: Ra and Ra + 8
    const uint32_t z_a = ptx::smem_u32(zsm), w_a = ptx::smem_u32(wsm);
    const int H8 = p.H >> 3;
    int st = 0; uint32_t ph = 0;
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const TileInfo ti = decode_tile(p, tile);
        if (!ti.valid) continue;
        // ---- z = tanh(enc + pred) of this warpgroup's 64 rows, 8 columns per item (the previous tile's MMAs have retired)
        for (int i = t128; i < 64 * H8; i += 128) {
            const int r = wg * 64 + i / H8, cc = i - (i / H8) * H8;
            const int t = ti.t0 + (r >> 3), u = ti.u0 + (r & 7);
            uint4 o = make_uint4(0u, 0u, 0u, 0u);
            if (t < ti.Tn && u < ti.Un) {
                const float4* pe = reinterpret_cast<const float4*>(p.enc + ((size_t)ti.b * p.maxT + t) * p.H + cc * 8);
                const float4* pq = reinterpret_cast<const float4*>(p.pred + ((size_t)ti.b * p.maxU + u) * p.H + cc * 8);
                const float4 e0 = __ldg(pe), e1 = __ldg(pe + 1), q0 = __ldg(pq), q1 = __ldg(pq + 1);
                o.x = ptx::pack_f16x2(ptx::tanh_approx(e0.x + q0.x), ptx::tanh_approx(e0.y + q0.y));
                o.y = ptx::pack_f16x2(ptx::tanh_approx(e0.z + q0.z), ptx::tanh_approx(e0.w + q0.w));
                o.z = ptx::pack_f16x2(ptx::tanh_approx(e1.x + q1.x), ptx::tanh_approx(e1.y + q1.y));
                o.w = ptx::pack_f16x2(ptx::tanh_approx(e1.z + q1.z), ptx::tanh_approx(e1.w + q1.w));
            }
            ptx::sts128(z_a + (uint32_t)((cc >> 3) * 16384 + r * 128 + (((cc & 7) ^ (r & 7)) << 4)), o);
        }
        ptx::fence_proxy_async_smem();
        ptx::named_bar_sync(1 + wg, 128);

        const int tslot = p.slot ? p.slot[tile] : tile;             // row block of this tile in the kept arrays
        const bool has_slot = tslot >= 0;       // false only when the caller's valid_tile_bound was too small (flagged by tile_compact_kernel)
        const size_t rowbase = (size_t)(has_slot ? tslot : 0) * 128;
        int lab[2];
        bool rv[2];
#pragma unroll
        for (int ri = 0; ri < 2; ++ri) {
            const int r = Ra + 8 * ri, t = ti.t0 + (r >> 3), u = ti.u0 + (r & 7);
            rv[ri] = t < ti.Tn && u < ti.Un;
            lab[ri] = (rv[ri] && u < ti.Un - 1) ? p.labels[(size_t)ti.b * (p.maxU - 1) + u] : -1;
        }
        float m2[2] = {-CUDART_INF_F, -CUDART_INF_F}, s[2] = {0.f, 0.f}, yb[2] = {0.f, 0.f}, yl[2] = {0.f, 0.f}, ref[2] = {0.f, 0.f};
        const uint32_t za = z_a + (uint32_t)wg * 8192u;
        for (int c = 0; c < NCH; ++c) {
            float acc[32];
#pragma unroll
            for (int i = 0; i < 32; ++i) acc[i] = 0.f;
            int prev = -1;
            for (int kb = 0; kb < KB; ++kb) {
                ptx::mbar_wait(&full[st], ph);
                const uint64_t ad = ptx::gmma_desc_k_sw128(za + (uint32_t)kb * 16384u);
                const uint64_t bd = ptx::gmma_desc_k_sw128(w_a + (uint32_t)st * 8192u);
                ptx::wgmma_fence();
#pragma unroll
                for (int k = 0; k < 4; ++k) ptx::wgmma_m64n64_f16<0>(acc, ad + (uint64_t)(k * 2), bd + (uint64_t)(k * 2), 1u);
                ptx::wgmma_commit();
                ptx::wgmma_wait<1>();
                if (prev >= 0 && t128 == 0) ptx::mbar_arrive(&empty[prev]);   // the previous K block's MMAs have retired
                prev = st;
                if (++st == stages) { st = 0; ph ^= 1; }
            }
            ptx::wgmma_wait<0>();
            if (t128 == 0) ptx::mbar_arrive(&empty[prev]);
            ptx::fence_regs(acc);

            // ---- epilogue: thread holds rows Ra, Ra + 8 at columns col0 + 8 j + 2 q + e
            const int col0 = c * FWD_NC;
            float bv[16];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float2 b2 = __ldg(reinterpret_cast<const float2*>(p.bias + col0 + 8 * j + 2 * q));
                bv[2 * j] = b2.x * LOG2E; bv[2 * j + 1] = b2.y * LOG2E;
            }
#pragma unroll
            for (int ri = 0; ri < 2; ++ri) {
                float y[16];
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    y[2 * j] = fmaf(acc[4 * j + 2 * ri], LOG2E, bv[2 * j]);
                    y[2 * j + 1] = fmaf(acc[4 * j + 2 * ri + 1], LOG2E, bv[2 * j + 1]);
                }
                if (c == 0) {      // the row's reference: maximum of its first 32 logits (j < 4 of the four lanes of the quad)
                    float r0 = y[0];
#pragma unroll
                    for (int i = 1; i < 8; ++i) r0 = fmaxf(r0, y[i]);
                    r0 = fmaxf(r0, __shfl_xor_sync(0xffffffffu, r0, 1));
                    r0 = fmaxf(r0, __shfl_xor_sync(0xffffffffu, r0, 2));
                    ref[ri] = r0;
                }
                float gm = y[0];
#pragma unroll
                for (int i = 1; i < 16; ++i) gm = fmaxf(gm, y[i]);
                if (__any_sync(0xffffffffu, gm - ref[ri] > FWD_REBASE))      // never taken on ordinary inputs
                    ref[ri] = fwd_rebase<MODE>(gm, ref[ri], p.dl, has_slot ? (long long)(rowbase + Ra + 8 * ri) : -1LL, p.V, q, c);
                const float mn = fmaxf(m2[ri], gm);
                uint32_t o[8];
                float accr = 0.f;
#pragma unroll
                for (int i = 0; i < 16; i += 2) {
                    const float e0 = ptx::ex2_approx(y[i] - ref[ri]), e1 = ptx::ex2_approx(y[i + 1] - ref[ri]);
                    accr += e0 + e1;
                    if (MODE == 2) o[i >> 1] = ptx::pack_bf16x2(e0, e1);
                }
                // y - ref <= FWD_REBASE here, so accr is finite.  A lane whose logits all lie more than 2^126 below the
                // quad's reference has accr == 0 (ex2 flushes), and its share of the row sum is below 2^-126 of it:
                // the clamp keeps that product 0 instead of 0 * inf.  The rounding is spelled out (a rounded product, then
                // one fma) so that MODE 0 and MODE 2 cannot be contracted differently and keep identical sums.
                const float a = __fmul_rn(accr, ptx::ex2_approx(fminf(ref[ri] - mn, 126.f)));
                if (MODE == 2 && has_slot) {
                    uint32_t* dst = reinterpret_cast<uint32_t*>(p.dl + (rowbase + Ra + 8 * ri) * p.V + col0 + 2 * q);
#pragma unroll
                    for (int j = 0; j < 8; ++j) dst[4 * j] = o[j];
                }
                s[ri] = fmaf(s[ri], ptx::ex2_approx(m2[ri] - mn), a);
                m2[ri] = mn;
                // the blank and label logits: held by one lane of the quad, at a column index known only at run time
                const int db = p.blank - col0 - 2 * q, dlb = lab[ri] - col0 - 2 * q;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        if (db == 8 * j + e) yb[ri] = y[2 * j + e];
                        if (dlb == 8 * j + e) yl[ri] = y[2 * j + e];
                    }
                }
            }
        }
        // ---- combine the quad's partial sums; one lane per row writes the cell's outputs
#pragma unroll
        for (int ri = 0; ri < 2; ++ri) {
            float M = fmaxf(m2[ri], __shfl_xor_sync(0xffffffffu, m2[ri], 1));
            M = fmaxf(M, __shfl_xor_sync(0xffffffffu, M, 2));
            float S = s[ri] * ptx::ex2_approx(m2[ri] - M);
            S += __shfl_xor_sync(0xffffffffu, S, 1);
            S += __shfl_xor_sync(0xffffffffu, S, 2);
            float b_ = yb[ri] + __shfl_xor_sync(0xffffffffu, yb[ri], 1);
            b_ += __shfl_xor_sync(0xffffffffu, b_, 2);
            float l_ = yl[ri] + __shfl_xor_sync(0xffffffffu, yl[ri], 1);
            l_ += __shfl_xor_sync(0xffffffffu, l_, 2);
            const int r = Ra + 8 * ri, t = ti.t0 + (r >> 3), u = ti.u0 + (r & 7);
            if (q != 0) continue;
            if (MODE == 2 && has_slot) p.gm[rowbase + r] = ref[ri];     // the row's reference (log2 domain)
            if (rv[ri] && p.lse) {   // (lse == NULL: a backward-time recompute that only wants the kept activations)
                const float lse2 = M + log2f(S);
                const long long cell = ((long long)ti.b * p.maxT + t) * p.maxU + u;
                p.lse[cell] = lse2 * LN2;
                const long long k = sk_index(ti.b, t, u, p.maxU, p.SK);
                p.lpb[k] = (b_ - lse2) * LN2;
                if (u < ti.Un - 1) p.lpl[k] = (l_ - lse2) * LN2;
            }
        }
    }
}

template <int MODE>
inline rnntStatus_t fwd_launch(const FwdGeom& g, const CUtensorMap& tm, const JointTcParams& p, cudaStream_t s) {
    if (!tc_smem_optin(reinterpret_cast<const void*>(joint_fwd_kernel<MODE>))) return RNNT_STATUS_EXECUTION_FAILED;
    const int ntiles = p.nb * p.nTb * p.nUb;
    const int grid = ntiles < tc_num_sms() ? ntiles : tc_num_sms();
    ScopedTimer tmr(MODE == 0 ? "joint_fwd_kernel<fwd>" : "joint_fwd_kernel<fwd+keep>", s);
    joint_fwd_kernel<MODE><<<grid, FWD_THREADS, g.smem_bytes, s>>>(tm, p);
    return cudaGetLastError() == cudaSuccess ? RNNT_STATUS_SUCCESS : RNNT_STATUS_EXECUTION_FAILED;
}

}  // namespace rb
