// Residual vector quantizer with the nearest-codeword search on the tensor cores (wgmma m64n128k8 tf32,
// 3xTF32 split) and EXACT fp32 re-scoring of near-ties, all n_q stages in one kernel.
//
// Reference: DistributedResidualVectorQuantization.forward (eval) funcodec/modules/quantization/ddp_core_vq.py:367-418,
// EuclideanCodebook.quantize :180-188 (dist = -(|x|^2 - 2 x.C^T + |c|^2), first maximal index).
//
// A cluster of s CTAs (s in {1, 2, 4}) owns 128 frames (rows) for every stage; rank r scores the codeword tiles
// [r * n_nt / s, (r + 1) * n_nt / s) of each stage against all 128 rows.
//   * the residual lives in shared memory as the 3xTF32 operand itself: hi and lo slabs (4 chunks of 32 dims,
//     canonical SWIZZLE_128B K-major), and hi + lo == the fp32 residual EXACTLY, so no separate copy is kept; every rank
//     keeps its own copy and updates it with the same winners;
//   * per stage the rank's share of the [K][D] codebook streams through a shared-memory ring as pre-split, pre-swizzled
//     slab images (one cp.async.bulk per 128-codeword x 32-dim slab); the compute warpgroup produces dot[128 rows x 128
//     codewords] tiles in registers (two m64 halves, 48 chained MMAs per accumulator for D = 128), evaluates
//     t = (|x|^2 - 2*dot) + |c|^2 in the reference's fp32 order and keeps the two best (value, index) of every row it holds,
//     merged across the 4 threads that share a row ((value, index) order == the reference's first minimal index);
//   * with s > 1 each rank sends its per-row (best, runner-up) list to every peer through DSMEM, and every rank merges
//     the s lists in the same (value, index) order.  A codeword's dot product comes from the same MMA sequence whichever
//     rank computes it, and the lexicographic top-2 of a union of disjoint sets is the top-2 of their top-2s, so the
//     winners (and every output bit) do not depend on s;
//   * the tensor-core dot carries ~1e-5 absolute error, so whenever best and runner-up are closer than
//     RESCORE_TOL both are re-scored with the exact sequential-fp32 dot product of the SIMT kernel (rvq_simt.cu) and
//     compared with the first-index tie-break: decisions equal the fp32 path's unless three candidates fall inside
//     the tolerance band;
//   * dequantize + residual update (ddp_core_vq.py:407-408) re-split the residual in place; the quantized sum is
//     rebuilt afterwards from the codes by embed_sum_kernel in the reference's accumulation order.  Rank r stores the
//     codes, sub_quants and encoder output of rows [r * 128 / s, (r + 1) * 128 / s) of the tile.
// FLOPs per launch: 2 * rows * K * D * n_q (x3 tensor passes); bytes: rows*D*4 in, codes out -> tensor-bound.
#include <climits>
#include "common.cuh"
#include "kernels.h"
#include "tc_sm90.cuh"

namespace fcb {

using namespace tc;

constexpr int RQ_M = 128;           // rows per CTA
constexpr int RQ_N = RVQ_TC_N;      // codewords per MMA tile (measured: 64-wide tiles with a 4-deep ring are 35% slower)
constexpr int RQ_NB = 2;            // codebook slab ring depth
constexpr int RQ_THREADS = 160;     // compute warpgroup (wgmma issue, scoring, residual update), copy warp
constexpr int RQ_MAX_RANKS = 4;     // CTAs per cluster at most
constexpr int RQ_CAND_BYTES = 4 * RQ_M * 4;    // one rank's candidate list: v1[128], i1[128], v2[128], i2[128]
constexpr float RQ_RESCORE_TOL = 4e-3f;

struct RqSmem {
    int a_slab;        // bytes of one (hi or lo) chunk slab: 128 rows x 128 B
    int off_b, off_cc, off_xx, off_idx, off_cand, off_bar, total;
};

// s: CTAs per cluster.  Candidate lists [buffer][rank]: one buffer for s = 1, two (by stage parity) for s > 1.
__host__ __device__ inline RqSmem rq_layout(int D, int K, int s) {
    RqSmem L;
    const int n_chunks = D / 32;
    L.a_slab = RQ_M * 128;
    L.off_b = 2 * n_chunks * L.a_slab;                // A: [chunk][hi|lo]
    L.off_cc = L.off_b + RQ_NB * 2 * RQ_N * 128;      // B ring: [stage][hi|lo][128 x 128 B]
    L.off_xx = L.off_cc + K * 4;
    L.off_idx = L.off_xx + RQ_M * 4;
    L.off_cand = L.off_idx + RQ_M * 4;                // 16-byte aligned (bulk-copy source and destination)
    L.off_bar = (L.off_cand + (s > 1 ? 2 : 1) * s * RQ_CAND_BYTES + 15) & ~15;
    L.total = L.off_bar + 8 * (2 * RQ_NB + 2) + 16;
    return L;
}

__global__ void __launch_bounds__(RQ_THREADS, 1) rvq_tc_kernel(const RvqParams p) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int D = p.D, K = p.K, T = p.T;
    const int n_chunks = D / 32;
    const int n_nt = K / RQ_N;
    const int s = (int)cluster_nctarank(), rank = s > 1 ? (int)cluster_ctarank() : 0;
    const int n_loc = n_nt / s, nt0 = rank * n_loc;     // this rank's codeword tiles
    const int own_lo = rank * (RQ_M / s), own_hi = own_lo + RQ_M / s;   // tile rows whose outputs this rank stores
    const RqSmem L = rq_layout(D, K, s);
    const long long M = (long long)p.B * T;
    const long long row0 = (long long)(blockIdx.x / s) * RQ_M;

    uint8_t* smA = smem_raw;
    uint8_t* smB = smem_raw + L.off_b;
    float* cc_s = reinterpret_cast<float*>(smem_raw + L.off_cc);
    float* xx_s = reinterpret_cast<float*>(smem_raw + L.off_xx);
    int* idx_s = reinterpret_cast<int*>(smem_raw + L.off_idx);
    float* cand_s = reinterpret_cast<float*>(smem_raw + L.off_cand);
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem_raw + L.off_bar);
    uint64_t* b_full = bars;                    // [RQ_NB]
    uint64_t* b_empty = b_full + RQ_NB;         // [RQ_NB]
    uint64_t* c_full = b_empty + RQ_NB;         // [2] the peers' candidate lists of a stage have landed (s > 1)

    if (tid == 0) {
        for (int i = 0; i < RQ_NB; ++i) { mbar_init(b_full + i, 1); mbar_init(b_empty + i, 1); }
        for (int i = 0; i < 2; ++i) mbar_init(c_full + i, 1);
        mbar_fence_init();
    }
    if (s > 1) cluster_sync(); else __syncthreads();    // the peers' barriers are initialised before any copy targets them
    const long long slab_bytes = 2LL * RQ_N * 128;      // one (n-tile, chunk) hi+lo image

    if (warp < 4) {
        const int jchunk = tid & 7, rsub = tid >> 3;    // (row, 16-byte chunk) mapping: 16 rows per pass
        // ---- load the encoder output (GroupNorm applied on load) into the hi/lo slabs
        for (int ch = 0; ch < n_chunks; ++ch) {
            uint8_t* hi = smA + (2 * ch) * L.a_slab;
            uint8_t* lo = hi + L.a_slab;
            for (int r = rsub; r < RQ_M; r += 16) {
                const long long row = row0 + r;
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                const int d = ch * 32 + jchunk * 4;
                if (row < M) {
                    const int b = (int)(row / T), t = (int)(row - (long long)b * T);
                    v = __ldg(reinterpret_cast<const float4*>(p.in.x + (long long)b * p.in.clip_stride + (long long)(p.in.row_off + t) * D + d));
                    if (p.in.stats) {
                        const float mean = p.in.stats[2 * b], rstd = p.in.stats[2 * b + 1];
                        const float4 g4 = __ldg(reinterpret_cast<const float4*>(p.in.gamma + d));
                        const float4 b4 = __ldg(reinterpret_cast<const float4*>(p.in.beta + d));
                        float a;
                        a = rstd * g4.x; v.x = fmaf(v.x, a, b4.x - a * mean);
                        a = rstd * g4.y; v.y = fmaf(v.y, a, b4.y - a * mean);
                        a = rstd * g4.z; v.z = fmaf(v.z, a, b4.z - a * mean);
                        a = rstd * g4.w; v.w = fmaf(v.w, a, b4.w - a * mean);
                    }
                    if (p.enc_out && r >= own_lo && r < own_hi) *reinterpret_cast<float4*>(p.enc_out + row * D + d) = v;
                }
                float4 h, l;
                split_tf32(v.x, h.x, l.x); split_tf32(v.y, h.y, l.y); split_tf32(v.z, h.z, l.z); split_tf32(v.w, h.w, l.w);
                const uint32_t o = (uint32_t)r * 128u + (uint32_t)((jchunk ^ (r & 7)) << 4);
                *reinterpret_cast<float4*>(hi + o) = h;
                *reinterpret_cast<float4*>(lo + o) = l;
            }
        }
        const int myrow = tid;                              // row of this thread for the re-scoring and the code store
        const bool own_row = myrow >= own_lo && myrow < own_hi;
        const uint32_t a_base = smem_u32(smA), b_base = smem_u32(smB);
        long long it = 0;                                   // codebook slab counter (the copy warp's order)
        auto lex_lt = [](float va, int ia, float vb, int ib) { return va < vb || (va == vb && ia < ib); };
        // (v1, i1, v2, i2) <- the two best of itself and the disjoint pair (ov1, oi1, ov2, oi2), both in (value, index) order
        auto merge2 = [&](float& v1, int& i1, float& v2, int& i2, float ov1, int oi1, float ov2, int oi2) {
            if (lex_lt(ov1, oi1, v1, i1)) {
                if (lex_lt(ov2, oi2, v1, i1)) { v2 = ov2; i2 = oi2; }
                else { v2 = v1; i2 = i1; }
                v1 = ov1; i1 = oi1;
            } else if (lex_lt(ov1, oi1, v2, i2)) {
                v2 = ov1; i2 = oi1;
            }
        };
        for (int q = 0; q < p.n_q; ++q) {
            const float* E = p.embed + (long long)q * K * D;
            // Candidate buffer of this stage.  With s > 1 a peer writes this buffer again at stage q + 2 only after it
            // received this rank's list of stage q + 1, which this rank sends after it has read the buffer (merge below)
            // and after its c_full phase of stage q has completed; the same chain orders the reuse of this rank's own
            // list as the source of its copies.
            const int cb = s > 1 ? (q & 1) : 0;
            float* cand_cb = cand_s + cb * s * (4 * RQ_M);
            // ---- |x|^2 in the SIMT kernel's order (8 lanes per row, stride-8 dims, xor-shuffle 1,2,4) and |c|^2
            asm volatile("bar.sync 1, 128;" ::: "memory");    // previous stage's residual update is complete
            if (s > 1 && tid == 0) mbar_arrive_expect_tx(c_full + cb, (uint32_t)((s - 1) * RQ_CAND_BYTES));
            for (int r = rsub; r < RQ_M; r += 16) {
                float sum = 0.f;
                for (int d = jchunk; d < D; d += 8) {
                    const uint32_t o = (uint32_t)r * 128u + (uint32_t)((((d & 31) >> 2) ^ (r & 7)) << 4) + (uint32_t)((d & 3) << 2);
                    const uint8_t* hi = smA + (2 * (d >> 5)) * L.a_slab;
                    const float v = *reinterpret_cast<const float*>(hi + o) + *reinterpret_cast<const float*>(hi + L.a_slab + o);
                    sum = fmaf(v, v, sum);
                }
                sum += __shfl_xor_sync(0xffffffffu, sum, 1);
                sum += __shfl_xor_sync(0xffffffffu, sum, 2);
                sum += __shfl_xor_sync(0xffffffffu, sum, 4);
                if (jchunk == 0) xx_s[r] = sum;
            }
            for (int c = tid; c < K; c += 128) cc_s[c] = __ldg(p.cnorm + (long long)q * K + c);
            fence_proxy_async_smem();                         // slabs of this stage are final -> visible to the wgmma
            asm volatile("bar.sync 1, 128;" ::: "memory");
            const float xx = xx_s[myrow];
            // accumulator rows of this thread: 64*h + 16*warp + lane/4 + 8*e (h: 64-row half, e: fragment row), k = 2*h + e;
            // best / runner-up per row as (value, index), index INT_MAX = none yet
            float xr[4], bv1[4], bv2[4];
            int bi1[4], bi2[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                xr[k] = xx_s[64 * (k >> 1) + 16 * warp + (lane >> 2) + 8 * (k & 1)];
                bv1[k] = 3.402823466e38f; bv2[k] = 3.402823466e38f;
                bi1[k] = INT_MAX; bi2[k] = INT_MAX;
            }
            for (int nt = nt0; nt < nt0 + n_loc; ++nt) {
                float acc0[RQ_N / 2], acc1[RQ_N / 2];
                int prev = -1;
                for (int ch = 0; ch < n_chunks; ++ch, ++it) {
                    const int bs = (int)(it % RQ_NB);
                    mbar_wait(b_full + bs, (uint32_t)((it / RQ_NB) & 1));
                    const uint32_t a_hi0 = a_base + (2 * ch) * L.a_slab, a_lo0 = a_hi0 + L.a_slab;
                    const uint32_t b_hi0 = b_base + bs * (uint32_t)slab_bytes, b_lo0 = b_hi0 + RQ_N * 128;
                    wgmma_fence();
#pragma unroll
                    for (int ks = 0; ks < 4; ++ks) {
                        const uint64_t db_hi = make_desc_k_sw128(b_hi0 + ks * 32), db_lo = make_desc_k_sw128(b_lo0 + ks * 32);
                        const uint32_t accum = (ch | ks) != 0;
                        // rows 0-63, then rows 64-127 (64 rows x 128 B further into the slab)
                        wgmma_m64n128k8_tf32(acc0, make_desc_k_sw128(a_lo0 + ks * 32), db_hi, accum);
                        wgmma_m64n128k8_tf32(acc0, make_desc_k_sw128(a_hi0 + ks * 32), db_lo, 1);
                        wgmma_m64n128k8_tf32(acc0, make_desc_k_sw128(a_hi0 + ks * 32), db_hi, 1);
                        wgmma_m64n128k8_tf32(acc1, make_desc_k_sw128(a_lo0 + 8192 + ks * 32), db_hi, accum);
                        wgmma_m64n128k8_tf32(acc1, make_desc_k_sw128(a_hi0 + 8192 + ks * 32), db_lo, 1);
                        wgmma_m64n128k8_tf32(acc1, make_desc_k_sw128(a_hi0 + 8192 + ks * 32), db_hi, 1);
                    }
                    wgmma_commit();
                    wgmma_wait<1>();                           // the previous slab has been read
                    if (prev >= 0 && tid == 0) mbar_arrive(b_empty + prev);
                    prev = bs;
                }
                wgmma_wait<0>();
                reg_fence(acc0);
                reg_fence(acc1);
                if (tid == 0) mbar_arrive(b_empty + prev);
                // every thread sees the columns of its rows in ascending order: strict '<' keeps the first minimal index
                auto scan = [&](const float (&a)[RQ_N / 2], int h) {
#pragma unroll
                    for (int j = 0; j < RQ_N / 8; ++j)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int k = 2 * h + e;
#pragma unroll
                            for (int x = 0; x < 2; ++x) {
                                const int c = nt * RQ_N + 8 * j + 2 * (lane & 3) + x;
                                const float tv = __fadd_rn(__fsub_rn(xr[k], 2.0f * a[4 * j + 2 * e + x]), cc_s[c]);
                                if (tv < bv1[k]) { bv2[k] = bv1[k]; bi2[k] = bi1[k]; bv1[k] = tv; bi1[k] = c; }
                                else if (tv < bv2[k]) { bv2[k] = tv; bi2[k] = c; }
                            }
                        }
                };
                scan(acc0, 0);
                scan(acc1, 1);
            }
            // merge the (disjoint, ascending-scanned) candidate pairs of the 4 threads sharing a row in (value, index) order
            // into this rank's list
            float* own = cand_cb + rank * (4 * RQ_M);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
#pragma unroll
                for (int o = 1; o <= 2; o <<= 1) {
                    const float ov1 = __shfl_xor_sync(0xffffffffu, bv1[k], o), ov2 = __shfl_xor_sync(0xffffffffu, bv2[k], o);
                    const int oi1 = __shfl_xor_sync(0xffffffffu, bi1[k], o), oi2 = __shfl_xor_sync(0xffffffffu, bi2[k], o);
                    merge2(bv1[k], bi1[k], bv2[k], bi2[k], ov1, oi1, ov2, oi2);
                }
                if ((lane & 3) == 0) {
                    const int rr = 64 * (k >> 1) + 16 * warp + (lane >> 2) + 8 * (k & 1);
                    own[rr] = bv1[k]; reinterpret_cast<int*>(own)[RQ_M + rr] = bi1[k];
                    own[2 * RQ_M + rr] = bv2[k]; reinterpret_cast<int*>(own)[3 * RQ_M + rr] = bi2[k];
                }
            }
            if (s > 1) {
                fence_proxy_async_smem();                     // the list -> visible to the bulk copies
                asm volatile("bar.sync 1, 128;" ::: "memory");
                if (tid == 0) {
                    for (int j = 1; j < s; ++j) {
                        const uint32_t peer = (uint32_t)((rank + j) % s);
                        bulk_s2peer(mapa_shared(smem_u32(own), peer), own, (uint32_t)RQ_CAND_BYTES, mapa_shared(smem_u32(c_full + cb), peer));
                    }
                }
                mbar_wait_cluster_backoff(c_full + cb, (uint32_t)((q >> 1) & 1), 32);
            } else {
                asm volatile("bar.sync 1, 128;" ::: "memory");
            }
            // this row's best / runner-up over all ranks' lists; a row without any finite score (NaN input) keeps index 0
            // and no runner-up, like the reference's max()
            float v1 = 3.402823466e38f, v2 = 3.402823466e38f;
            int i1 = INT_MAX, i2 = INT_MAX;
            for (int r = 0; r < s; ++r) {
                const float* l = cand_cb + r * (4 * RQ_M);
                merge2(v1, i1, v2, i2, l[myrow], reinterpret_cast<const int*>(l)[RQ_M + myrow], l[2 * RQ_M + myrow],
                       reinterpret_cast<const int*>(l)[3 * RQ_M + myrow]);
            }
            if (i1 == INT_MAX) i1 = 0;
            if (i2 == INT_MAX) i2 = -1;
            // ---- exact fp32 re-scoring of near-ties (sequential fmaf chain == rvq_simt.cu)
            int best = i1;
            if (row0 + myrow < M && v2 - v1 < RQ_RESCORE_TOL + 2e-5f * fabsf(v1) && i2 >= 0) {
                float d1 = 0.f, d2 = 0.f;
                const float* c1 = E + (long long)i1 * D;
                const float* c2 = E + (long long)i2 * D;
                for (int d = 0; d < D; ++d) {
                    const uint32_t o = (uint32_t)myrow * 128u + (uint32_t)((((d & 31) >> 2) ^ (myrow & 7)) << 4) + (uint32_t)((d & 3) << 2);
                    const uint8_t* hi = smA + (2 * (d >> 5)) * L.a_slab;
                    const float x = *reinterpret_cast<const float*>(hi + o) + *reinterpret_cast<const float*>(hi + L.a_slab + o);
                    d1 = fmaf(x, __ldg(c1 + d), d1);
                    d2 = fmaf(x, __ldg(c2 + d), d2);
                }
                const float t1 = __fadd_rn(__fsub_rn(xx, 2.0f * d1), cc_s[i1]);
                const float t2 = __fadd_rn(__fsub_rn(xx, 2.0f * d2), cc_s[i2]);
                if (t2 < t1 || (t2 == t1 && i2 < i1)) best = i2;
            }
            idx_s[myrow] = best;
            if (row0 + myrow < M && own_row) p.codes[(long long)q * M + row0 + myrow] = (long long)best;
            asm volatile("bar.sync 1, 128;" ::: "memory");
            // ---- dequantize + residual update (all wgmma of the stage have completed).
            // 8 passes of 16 rows; the codeword reads of pass i+1 (L2 latency) are in flight while pass i is re-split.
            {
                constexpr int MAXCH = 4;                       // D <= 128 on this path
                float4 cv[MAXCH], nv[MAXCH];
                auto load_c = [&](int r, float4 (&dst)[MAXCH]) {
#pragma unroll
                    for (int ch = 0; ch < MAXCH; ++ch) {
                        dst[ch] = make_float4(0.f, 0.f, 0.f, 0.f);
                        if (ch < n_chunks && row0 + r < M)
                            dst[ch] = __ldg(reinterpret_cast<const float4*>(E + (long long)idx_s[r] * D + ch * 32 + jchunk * 4));
                    }
                };
                load_c(rsub, cv);
                for (int r = rsub; r < RQ_M; r += 16) {
                    if (r + 16 < RQ_M) load_c(r + 16, nv);
                    const long long row = row0 + r;
                    if (row < M) {
                        const uint32_t o = (uint32_t)r * 128u + (uint32_t)((jchunk ^ (r & 7)) << 4);
#pragma unroll
                        for (int ch = 0; ch < MAXCH; ++ch) {
                            if (ch < n_chunks) {
                                uint8_t* hi = smA + (2 * ch) * L.a_slab;
                                uint8_t* lo = hi + L.a_slab;
                                const float4 h0 = *reinterpret_cast<const float4*>(hi + o);
                                const float4 l0 = *reinterpret_cast<const float4*>(lo + o);
                                const float4 c4 = cv[ch];
                                float4 x;
                                x.x = (h0.x + l0.x) - c4.x; x.y = (h0.y + l0.y) - c4.y; x.z = (h0.z + l0.z) - c4.z; x.w = (h0.w + l0.w) - c4.w;
                                float4 h, l;
                                split_tf32(x.x, h.x, l.x); split_tf32(x.y, h.y, l.y); split_tf32(x.z, h.z, l.z); split_tf32(x.w, h.w, l.w);
                                *reinterpret_cast<float4*>(hi + o) = h;
                                *reinterpret_cast<float4*>(lo + o) = l;
                                if (p.sub_quants && r >= own_lo && r < own_hi) {
                                    const int b = (int)(row / T), t = (int)(row - (long long)b * T);
                                    const int d = ch * 32 + jchunk * 4;
                                    float* sq = p.sub_quants + (((long long)q * p.B + b) * D + d) * T + t;
                                    sq[0] = c4.x; sq[(long long)T] = c4.y; sq[2LL * T] = c4.z; sq[3LL * T] = c4.w;
                                }
                            }
                        }
                    }
#pragma unroll
                    for (int ch = 0; ch < MAXCH; ++ch) cv[ch] = nv[ch];
                }
            }
        }
    } else if (warp == 4) {
        // =========================================================== this rank's codebook slabs via the bulk-copy engine
        if (lane == 0) {
            long long it = 0;
            for (int q = 0; q < p.n_q; ++q) {
                const uint8_t* qbase = reinterpret_cast<const uint8_t*>(p.embed_tc) + (long long)q * n_nt * n_chunks * slab_bytes;
                for (int nt = nt0; nt < nt0 + n_loc; ++nt)
                    for (int ch = 0; ch < n_chunks; ++ch, ++it) {
                        const int bs = (int)(it % RQ_NB);
                        mbar_wait_backoff(b_empty + bs, (uint32_t)((it / RQ_NB) & 1) ^ 1, 64);
                        mbar_arrive_expect_tx(b_full + bs, (uint32_t)slab_bytes);
                        bulk_g2s(smB + bs * slab_bytes, qbase + ((long long)nt * n_chunks + ch) * slab_bytes, (uint32_t)slab_bytes, b_full + bs);
                    }
            }
        }
    }
    if (s > 1) cluster_sync();    // no CTA exits while a peer's copy may still read or write its shared memory
}

bool rvq_tc_supported(int D, int K) {
    return D % 32 == 0 && D >= 32 && D <= 128 && K % RQ_N == 0 && rq_layout(D, K, 1).total <= 225 * 1024;
}

// Clusters of s CTAs (index: s / 2 - 1 for s = 2, 4) that a device holds at once at 225 KB of shared memory each, the most
// the kernel asks for, so the count holds for every shape; per device ordinal (ordinals beyond the table are queried at
// every launch)
constexpr int RQ_DEVICES = 64;
static int g_rq_max_clusters[RQ_DEVICES][2] = {};

cudaError_t launch_rvq_tc(const RvqParams& p, cudaStream_t st) {
    if (!rvq_tc_supported(p.D, p.K) || !p.embed_tc) return cudaErrorInvalidValue;
    {
        cudaError_t e = ensure_dynamic_smem((const void*)rvq_tc_kernel, 225 * 1024);
        if (e != cudaSuccess) return e;
    }
    const long long M = (long long)p.B * p.T;
    const long long tiles = (M + RQ_M - 1) / RQ_M;
    // The largest s in {4, 2} that divides the codeword tiles and whose clusters for all row tiles fit in one wave: a
    // second wave would take longer than s = 1, where every row tile has an SM of its own.
    for (int s = RQ_MAX_RANKS; s > 1; s >>= 1) {
        if ((p.K / RQ_N) % s != 0 || rq_layout(p.D, p.K, s).total > 225 * 1024) continue;
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeClusterDimension;
        attr[0].val.clusterDim.x = (unsigned)s; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
        cudaLaunchConfig_t cfg = {};
        cfg.blockDim = dim3(RQ_THREADS);
        cfg.stream = st;
        cfg.attrs = attr;
        cfg.numAttrs = 1;
        int dev = 0;
        cudaError_t e = cudaGetDevice(&dev);
        if (e != cudaSuccess) return e;
        int max_clusters = dev < RQ_DEVICES ? g_rq_max_clusters[dev][s / 2 - 1] : 0;
        if (max_clusters == 0) {
            cfg.gridDim = dim3((unsigned)s);
            cfg.dynamicSmemBytes = 225 * 1024;
            e = cudaOccupancyMaxActiveClusters(&max_clusters, rvq_tc_kernel, &cfg);
            if (e != cudaSuccess) return e;
            if (max_clusters < 1) max_clusters = -1;    // cached as "none"
            if (dev < RQ_DEVICES) g_rq_max_clusters[dev][s / 2 - 1] = max_clusters;
        }
        if (tiles > max_clusters) continue;
        cfg.gridDim = dim3((unsigned)(tiles * s));
        cfg.dynamicSmemBytes = rq_layout(p.D, p.K, s).total;
        return cudaLaunchKernelEx(&cfg, rvq_tc_kernel, p);
    }
    rvq_tc_kernel<<<(unsigned)tiles, RQ_THREADS, rq_layout(p.D, p.K, 1).total, st>>>(p);
    return cudaGetLastError();
}

}  // namespace fcb
