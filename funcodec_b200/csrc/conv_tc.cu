// Implicit-GEMM Conv1d on the Hopper tensor cores (wgmma m64nNk16, fp16 operands in shared memory, fp32 accumulators in
// registers), fp32-faithful through a 3-term FP16 split: both operands are pre-scaled by a power of two (activations x16, weights
// per layer so that max|w| lands in [2^13, 2^14)), x = hi + lo with hi = fp16(x), lo = fp16(x - hi), and
// D += lo*hi + hi*lo + hi*hi in fp32; the epilogue multiplies by the (exact) inverse scale.  Same accuracy as a 3xTF32 split
// (both drop the lo*lo term, ~2^-22 relative), at twice the tensor throughput and half the shared-memory operand bytes per
// MAC (K = 16 per MMA instead of 8; a 128-byte swizzle row holds 64 channels).
//
// Same contract as conv_simt.cu (fused [GroupNorm apply + resblock add + ELU + reflect pad] on the input,
// bias + raw store + GroupNorm partial statistics on the output), reference semantics
// funcodec/modules/normed_modules/conv.py:243-261 / :281-305.
//
// GEMM view (channels-last makes both operands K-major):
//     D[t (M = 128 time rows), co (N = n_tile)] = sum_{tap k} sum_{ci} X[t*S + k - pad_l][ci] * W[k][ci][co]
//   * A (activations): one "unit" = (32-channel chunk, stride phase p): the rows {(t0+u)*S + p - pad_l}
//     are transformed by a producer group and written (hi and lo slabs) into the canonical SWIZZLE_128B
//     K-major layout; a ring stage holds a 64-channel chunk, i.e. two units side by side (with two producer groups each
//     fills one half, a single group fills half 0 then half 1; layers with a single 32-channel chunk fill half a stage
//     and the groups alternate stages);
//     every tap k = q*S + p of that phase is then just a ROW-SHIFTED view (start address
//     + q*128 B; the hardware swizzle works on absolute address bits) of the same slab -- no im2col copy.
//   * B (weights): pre-split, pre-swizzled slab images in HBM (engine.cu pack_tc), one cp.async.bulk
//     (TMA engine, 1-D) per (chunk, tap) into a ring, completion on an mbarrier.
//   * PERSISTENT CTAs (one per SM) walk a static list of (clip, n-tile, time-tile) tiles; every role keeps
//     running across tile boundaries, so the next tile's loads overlap the previous tile's MMAs and epilogue.
//   * warp roles (every role fills whole warpgroups and sets its own register budget with setmaxnreg at entry; TcRoles):
//     first the producer groups -- two at N_TILE <= 64 (5 warpgroups, 640 threads: two units of global loads in flight, for
//     the HBM-bound shallow layers), one at N_TILE = 128 (4 warpgroups, 512 threads: its registers go to the consumers'
//     128-column accumulators); then the control warpgroup: warp 0 weight copies, warp 1 raw-tile TMA loads, warps 2-3
//     idle; then the two consumer warpgroups, each issuing the wgmma of 64 of the 128 tile rows (its A view starts 64 rows
//     further into the stage) and running the epilogue of its rows.  A consumer issues a tap's 12 (or 6) wgmma back to back
//     as one commit group, from uniform control flow, and touches its accumulators only after the group's final wait.
//   * N_TILE = 128 (1-D layers with C_out % 128 == 0) transforms each activation element once per 128 output columns instead
//     of once per 64; its epilogue still writes one GroupNorm partial per 64 columns, at the index a 64-column tile would
//     use, so the statistics (and every output bit) do not depend on the tile width.
//   * 2-CTA pairs (PAIR, 1-D N_TILE = 128 layers on the raw ring with an even number of n-tiles): a cluster's two CTAs take
//     n-tiles 2j and 2j + 1 of one time tile, whose A stages are identical.  Each fetches and transforms half of the slab rows and
//     copies them into the peer's stage (cp.async.bulk shared::cta -> shared::cluster, completing on the peer's a_full); each
//     consumer warpgroup releases a stage in both CTAs.  Weights, MMA issue and epilogue are those of the single-CTA kernel.
//   * the tensor core adds into its fp32 accumulator with truncation, so a long chain loses ~1 ulp per MMA:
//     chains are cut every ~48 MMAs and each finished group is folded into running totals (registers) with
//     round-to-nearest CUDA-core adds; the epilogue (bias, channels-last store, GroupNorm partial sums) reads the totals.
// Roofline: tensor pipe (3 MMAs per fp32-equivalent product) for the deep layers; HBM for the C <= 64 layers.
//
// FREQ = true is the FreqCodec 2-D mode (SConv2d / SConvTranspose2d, conv.py:317-447): a "clip" of the tile list is a
// pseudo-clip (clip b, output frequency row f_out) and the gathered input channel cg = kf*cin + c of a chunk comes from
// frequency row f_out*SF + kf - pad_f (reflect / zero indexed) of the [B][F][T][cin] input, so a 32-channel chunk holds
// 32/cin frequency taps (cin < 32) or a 32-channel slice of one tap; everything downstream of the producers (weight
// slabs [tap kt][cg][co], MMA issue, folding) is the 1-D machinery.  The epilogue scatters the phases of a transposed
// conv (co -> (pf, pt, channel)) and can store fewer channels than the padded n-tile (the 32 -> 3 output conv).
#include <cuda.h>
#include "common.cuh"
#include "kernels.h"
#include "tc_sm90.cuh"
#include <stdlib.h>
#include <type_traits>

namespace fcb {

using namespace tc;

constexpr int TC_M = 128;          // time rows per tile
constexpr int TC_KC = 32;          // channels per producer unit (half of a 128-byte fp16 swizzle row)
constexpr int TC_RAW_MAX = 8;      // raw activation ring (TMA-staged units): at most 8 slots
constexpr int TC_PROD = 128;       // producer threads per group (one warpgroup, one unit)
constexpr int TC_PROWS = TC_PROD / 8;   // rows per producer pass (8 threads x 4 channels cover a row's 32 channels)
constexpr int TC_A_ROWS_MAX = 144; // A slab rows: 128 + (K - 1) / S <= 16 (conv_tc_supported), rounded up to 8
constexpr int TC_GROUP_MMAS = 48;  // target number of wgmma chained in one accumulator before the fp32 fold
// Warp layout and per-thread register budgets (setmaxnreg) of one tile width, all compile-time.  Every role fills whole
// warpgroups: PROD_GROUPS producer warpgroups, then the control warpgroup, then the two consumer warpgroups.  The launch gives
// every thread LAUNCH_REGS (the CTA's pool is THREADS x LAUNCH_REGS), which the roles split among themselves:
//   * N_TILE <= 64: 5 warpgroups (640 threads x 96 = 61 440): producers 2 x 96, control 64, consumers 2 x 112.  A consumer holds
//     N_TILE / 2 accumulators plus as many running totals (64 at N_TILE = 64); the shallow (C <= 64) layers are latency- and
//     HBM-bound and need both producer groups' loads in flight.
//   * N_TILE = 128: 4 warpgroups (512 threads x 128 = 65 536): one producer group at 112 fills both 32-channel halves of every
//     stage, control 64, consumers 2 x 168 (64 accumulators + 64 running totals).  Each transformed element now feeds 128
//     columns, so one producer group carries as much transform work per MAC as two did at N_TILE = 64.
// Each budget is spill-free as compiled (ptxas is not monotonic in them: pick them by compiling); a producer keeps three passes
// of row loads in flight on the edge path, and the raw-tile TMA warp needs more than 32.
template <int N_TILE>
struct TcRoles {
    static constexpr int PROD_GROUPS = N_TILE > 64 ? 1 : 2;
    static constexpr int THREADS = 128 * (PROD_GROUPS + 3);
    static constexpr int LAUNCH_REGS = 65536 / THREADS / 8 * 8;
    static constexpr int PROD_REGS = N_TILE > 64 ? 112 : 96, CTL_REGS = 64, CONS_REGS = N_TILE > 64 ? 168 : 112;
    static constexpr int CTL_WG = PROD_GROUPS;            // warpgroup of the control role; the consumers follow it
    static constexpr int CONS_WG = PROD_GROUPS + 1;
    // GroupNorm partials per tile: one per 64 columns, so a layer's partial count and fp64 reduction order do not depend on the
    // tile width
    static constexpr int PARTS = N_TILE > 64 ? N_TILE / 64 : 1;
    static_assert(128 * (2 * CONS_REGS + PROD_GROUPS * PROD_REGS + CTL_REGS) <= THREADS * LAUNCH_REGS, "register pool");
};

// ELU with the hardware exponential (ex2.approx): |error| <= ~2e-7 on the (0, 1] range of exp(x), the same order as
// one fp32 rounding of the reference's exp(x) - 1.  (The SIMT path keeps expf.)
__device__ __forceinline__ float elu_fast(float v) { return v > 0.f ? v : (__expf(v) - 1.0f); }
// the same on a value pre-multiplied by the operand scale s (a power of two): s*elu(v) from vs = s*v with k = log2(e)/s.
// Scaling by a power of two commutes with every rounding involved, so this equals s * elu_fast(v) bit for bit.
__device__ __forceinline__ float elu_scaled(float vs, float k, float s) { return vs > 0.f ? vs : fmaf(exp2f_approx(vs * k), s, -s); }

struct TcSmemLayout {
    int a_rows;        // rows per A slab (multiple of 8)
    int a_stage;       // bytes per A stage (hi + lo)
    int b_stage;       // bytes per B stage (hi + lo)
    int na, nb;        // ring depths
    int nraw, raw_slot, raw_in1, raw_cf;   // raw activation ring: slots, bytes per slot, offsets of in1 / coefficients in a slot
    int off_b, off_raw, off_bar, total;
};

// A slab rows a CTA transforms and its raw boxes hold: all a_rows, or in a 2-CTA pair the share of rank 0 (rows [0, share)), rank 1
// taking the rest; a multiple of 8 rows keeps both shares whole swizzle groups
__host__ __device__ inline int tc_raw_rows(int a_rows, bool pair) { return pair ? ((a_rows / 2 + 7) / 8) * 8 : a_rows; }

__host__ __device__ inline TcSmemLayout tc_layout(int K, int S, int n_tile, int na, int nb, int nraw = 0, int raw_pitch = 128,
                                                   int has1 = 0, bool pair = false) {
    TcSmemLayout L;
    const int qmax = (K - 1) / S;
    L.a_rows = ((TC_M + qmax + 7) / 8) * 8;
    const int raw_rows = tc_raw_rows(L.a_rows, pair);
    L.a_stage = 2 * L.a_rows * 128;
    L.b_stage = 2 * n_tile * 128;
    L.na = na; L.nb = nb;
    L.off_b = na * L.a_stage;
    // raw slot: [in0 rows][in1 rows][a0 | b0 | a1 | b1 coefficient slices of the unit's 32 channels (4 x 128 B)]
    L.nraw = nraw;
    L.raw_in1 = raw_rows * raw_pitch;
    L.raw_cf = (1 + has1) * raw_rows * raw_pitch;
    L.raw_slot = (L.raw_cf + 512 + 127) / 128 * 128;
    L.off_raw = L.off_b + nb * L.b_stage;
    L.off_bar = L.off_raw + nraw * L.raw_slot;
    // + statistics scratch: [partials per tile][8 consumer warps][2] doubles + the finalisation flag
    L.total = L.off_bar + 8 * (2 * na + 2 * nb + 2 * TC_RAW_MAX) + 128 * (n_tile > 64 ? n_tile / 64 : 1) + 32;
    return L;
}

// ring stages (64-channel chunk, phase) chained in one accumulation group
__host__ __device__ inline int tc_units_per_group(int K, int S, int group_mmas) {
    const int taps = (K + S - 1) / S;                  // max taps of a phase
    int g = group_mmas / (12 * taps);
    return g < 1 ? 1 : g;
}

// Launch-invariant quantities computed on the host and read from the kernel-parameter constant bank (instead of being
// derived -- and kept live in registers -- by every thread).
struct TcArgs {
    TcSmemLayout L;
    int na, nb, n_tiles, w_resident, nraw;
    int n_chunks, n_sc, split, n_units, upg, n_groups, n_tt, n_nt, units_per_tile, tq_rows, raw_pitch;
    int raw_rows;      // tc_raw_rows
};

struct TcTile { int b, nt, tt; };

__device__ __forceinline__ TcTile tc_tile(int id, int n_nt, int n_tt) {
    TcTile t;
    t.nt = id % n_nt;                  // n-tile fastest: concurrent CTAs share the activation rows in L2
    const int r = id / n_nt;
    t.tt = r % n_tt;
    t.b = r / n_tt;
    return t;
}

// One tap of a stage as one commit group: KSTEPS k-steps of 16 channels, 3 wgmma each (lo*hi, hi*lo, hi*hi -- the k-order of
// every output column is fixed by this order).  `accum` = 0 starts a fresh accumulation group with the first MMA.
template <int N_TILE, int KSTEPS>
__device__ __forceinline__ void tc_issue_tap(float (&acc)[N_TILE / 2], uint32_t a_hi, uint32_t a_lo, uint32_t b_hi, uint32_t b_lo,
                                             uint32_t accum) {
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < KSTEPS; ++ks) {
        WgmmaF16<N_TILE>::mma(acc, make_desc_k_sw128(a_lo + ks * 32), make_desc_k_sw128(b_hi + ks * 32), ks == 0 ? accum : 1u);
        WgmmaF16<N_TILE>::mma(acc, make_desc_k_sw128(a_hi + ks * 32), make_desc_k_sw128(b_lo + ks * 32), 1u);
        WgmmaF16<N_TILE>::mma(acc, make_desc_k_sw128(a_hi + ks * 32), make_desc_k_sw128(b_hi + ks * 32), 1u);
    }
    wgmma_commit();
}

// PAIR (1-D, N_TILE = 128, raw ring, an even number of n-tiles; launched as 2-CTA clusters): the CTAs of a cluster take n-tiles
// 2j and 2j + 1 of the same (clip, time tile) -- the tile list puts n-tiles fastest and the grid is even, so the usual walk
// (blockIdx.x, stride gridDim.x) gives them that pairing at every step.  Their A stages are identical: cluster rank r fetches and
// transforms only its share of the slab rows (ka.raw_rows rows from r * ka.raw_rows) and copies them into the peer's stage.
template <int N_TILE, bool FREQ, bool PAIR = false>
__global__ void __launch_bounds__(TcRoles<N_TILE>::THREADS, 1) conv1d_tc_kernel(const __grid_constant__ ConvParams p, const __grid_constant__ TcArgs ka,
                                                                 const __grid_constant__ CUtensorMap tm0,
                                                                 const __grid_constant__ CUtensorMap tm1) {
    static_assert(!PAIR || (N_TILE == 128 && !FREQ), "pairs are built for the 1-D 128-column layout");
    using R = TcRoles<N_TILE>;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int C_in = p.C_in, K = p.K, S = p.S;
    const bool has1 = p.in1.x != nullptr;
    const TcSmemLayout& L = ka.L;
#define na_stages ka.na
#define nb_stages ka.nb
#define n_tiles ka.n_tiles
#define w_resident ka.w_resident
#define nraw ka.nraw
#define raw_pitch ka.raw_pitch              /* bytes per row of a raw (TMA-staged) unit */
#define n_chunks ka.n_chunks                /* 32-channel chunks; C_in = 16: one half-empty chunk (zero channels, zero weights) */
#define n_sc ka.n_sc                        /* 64-channel stage chunks */
#define n_units ka.n_units                  /* ring stages per tile */
#define upg ka.upg
#define n_groups ka.n_groups
#define n_tt ka.n_tt
#define n_nt ka.n_nt
    const bool split = ka.split != 0;                     // a stage holds two 32-channel units (halves)

    uint8_t* smA = smem_raw;
    uint8_t* smB = smem_raw + L.off_b;
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem_raw + L.off_bar);
    uint64_t* a_full = bars;                       // [na]   producer arrivals (128 per 32-channel half written)
    uint64_t* a_empty = a_full + na_stages;        // [na]   one arrival per consumer warpgroup (its wgmma have read the stage)
    uint64_t* b_full = a_empty + na_stages;        // [nb]   expect_tx
    uint64_t* b_empty = b_full + nb_stages;        // [nb]   one arrival per consumer warpgroup
    uint64_t* raw_full = b_empty + nb_stages;      // [TC_RAW_MAX] expect_tx (TMA tile + coefficient slices)
    uint64_t* raw_empty = raw_full + TC_RAW_MAX;   // [TC_RAW_MAX] 128 arrivals of the consuming producer group
    double* red = reinterpret_cast<double*>(raw_empty + TC_RAW_MAX);   // [PARTS][8][2] statistics scratch + finalisation flag
    uint8_t* smR = smem_raw + L.off_raw;
    // TMA-staged units (nraw > 0, 1-D layers): an INTERIOR tile needs only rows inside [0, rows covered by the tensor map) -- no
    // reflection, no zero padding -- so its units arrive as dense [a_rows][32 channel] boxes through the raw ring.  In a 1-D layer the
    // first / last tiles of a clip take the ring too: the box zero-fills the rows outside the input, and the producers apply the
    // per-thread path's index map to those rows (zero, or a reflected row read from global memory).  The 2-D mode keeps its edge
    // tiles on the per-thread global loads.  Units of a tile in ring order:
    // stage-major, half-minor; every role derives the slot from the same running count.
#define units_per_tile ka.units_per_tile
#define tq_rows ka.tq_rows                  /* rows per phase the tensor map exposes */
    auto tile_interior = [&](int t0) -> bool {
        if (nraw == 0) return false;
        // first / last input row that a VALID output row of the tile needs (a partial last tile only counts its real rows: the
        // rows a 1x1 layer does not have arrive zero-filled and feed discarded output rows only)
        const int t_last = (t0 + TC_M < p.T_out ? t0 + TC_M : p.T_out) - 1;
        const int lo = t0 * S - p.pad_l;
        const int hi = t_last * S - p.pad_l + (K - 1);
        return lo >= 0 && hi < tq_rows * S;
    };
    // tiles whose units come through the raw ring: every tile of a 1-D layer (an edge tile patches its padding rows per row, see the
    // producers), the interior tiles of a 2-D layer
    auto tile_raw = [&](int t0) -> bool { return FREQ ? tile_interior(t0) : nraw > 0; };

    // PAIR: a_full also takes one local arrival that posts the expect_tx of the rows the peer copies in; a_empty takes both CTAs'
    // consumer warpgroups, since a producer writes into both CTAs' stages
    const uint32_t rank = PAIR ? cluster_ctarank() : 0u, peer = rank ^ 1u;
    const int r0 = (int)rank * ka.raw_rows;                                         // first A slab row this CTA transforms
    const int r_end = PAIR ? min(L.a_rows, r0 + ka.raw_rows) : L.a_rows;
    if (tid == 0) {
        for (int i = 0; i < na_stages; ++i) {
            mbar_init(a_full + i, (split ? 2 * TC_PROD : TC_PROD) + (PAIR ? 1 : 0));
            mbar_init(a_empty + i, PAIR ? 4 : 2);
        }
        for (int i = 0; i < nb_stages; ++i) { mbar_init(b_full + i, 1); mbar_init(b_empty + i, 2); }
        for (int i = 0; i < TC_RAW_MAX; ++i) { mbar_init(raw_full + i, 1); mbar_init(raw_empty + i, TC_PROD); }
        mbar_fence_init();
    }
    // PAIR: no remote arrival or copy may reach a barrier of the peer before the peer has initialised it
    if (PAIR) cluster_sync(); else __syncthreads();

    const int role = warp >> 2;                     // warpgroup: producers, then control, then the two consumers
    if (role < R::PROD_GROUPS) {
        // =========================================================== producers: transformed A slabs
        setmaxnreg_dec<R::PROD_REGS>();
        const int grp = role;
        const int ptid = tid & (TC_PROD - 1);
        const int jchunk = ptid & 7;                // 4 channels (16 bytes of fp32 in HBM, 8 bytes of fp16 in the slab)
        // rows of a warp: {b, b+1, b+4, b+5}: its four 64-byte half rows land on all 32 banks (2 wavefronts per 8-byte store)
        const int wq = (ptid >> 5), lq = (lane >> 3);
        const int rsub = ((wq >> 1) << 3) + ((wq & 1) << 1) + (lq & 1) + ((lq >> 1) << 2);      // TC_PROWS = 16 rows per pass
        constexpr int NR = TC_A_ROWS_MAX / TC_PROWS;                                             // passes per unit
        // passes per raw unit: a PAIR CTA transforms at most half of the rows, rounded up to 8
        constexpr int NR_RAW = PAIR ? ((TC_A_ROWS_MAX / 2 + 7) / 8 * 8 + TC_PROWS - 1) / TC_PROWS : NR;
        auto wait_a_empty = [&](uint64_t* bar, uint32_t par) {
            if (PAIR) mbar_wait_cluster_backoff(bar, par, 64);       // the peer's consumers arrive on it too
            else if (p.dbg & 64) mbar_wait(bar, par);
            else mbar_wait_backoff(bar, par, 64);
        };
        // PAIR hand-off: this CTA's rows of the hi and lo slabs go to the same offsets in the peer's stage (the swizzle follows the
        // address, so a same-offset copy keeps the layout), completing on the peer's a_full
        const uint32_t hand_bytes = (uint32_t)(r_end - r0) * 128u;
        const uint32_t peer_bytes = 2u * (uint32_t)(L.a_rows - (r_end - r0)) * 128u;
        const uint32_t smA_peer = PAIR ? mapa_shared(smem_u32(smA), peer) : 0u;
        const uint32_t a_full_peer = PAIR ? mapa_shared(smem_u32(a_full), peer) : 0u;
        const int gt_max = (p.T_out - 1) * S - p.pad_l + (K - 1);
        // this group's cursor over the CTA's global stage sequence (tile-major).  split: every stage is filled by both groups
        // (group g writes the 32-channel half g), or by the single group, half 0 then half 1; otherwise (one 32-channel chunk)
        // the groups take alternate stages and the ring slot advances PROD_GROUPS at a time (na is even), so no division /
        // modulo is needed in the loop.  Every written half is one group's 128 arrivals on a_full.
        const int step = split ? 1 : R::PROD_GROUPS;
        const int half0 = (split && R::PROD_GROUPS == 2) ? grp : 0;
        int half = half0;
        int tile = blockIdx.x, unit = split ? 0 : grp;
        int as = unit % na_stages;
        uint32_t aphase = 0;
        const float in_scale = p.tc_in_scale;
        int rawbase = 0;                            // raw-ring units of the interior tiles this CTA has passed
        while (unit >= n_units && tile < n_tiles) {
            if (tile_raw(tc_tile(tile, n_nt, n_tt).tt * TC_M)) rawbase += units_per_tile;
            unit -= n_units; tile += gridDim.x;
        }
        while (tile < n_tiles) {
            const TcTile tl = tc_tile(tile, n_nt, n_tt);
            const int t0 = tl.tt * TC_M;
            int b = tl.b, f_out = 0;
            if (FREQ) { b = tl.b / p.fq.F_out; f_out = tl.b - b * p.fq.F_out; }
            const int pitch = FREQ ? p.fq.cin : C_in;          // channels per stored input row
            const float* x0 = p.in0.x + (long long)b * p.in0.clip_stride + (long long)p.in0.row_off * pitch;
            const float* x1 = has1 ? p.in1.x + (long long)b * p.in1.clip_stride + (long long)p.in1.row_off * pitch : nullptr;
            const float* cf0 = p.in0.coef ? p.in0.coef + (long long)b * 2 * pitch : nullptr;
            const float* cf1 = (has1 && p.in1.coef) ? p.in1.coef + (long long)b * 2 * pitch : nullptr;
            const int cur_tile = tile;
            const bool raw = tile_raw(t0);
            const bool edge = !FREQ && raw && !tile_interior(t0);   // raw-staged edge tile (1-D): padding rows patched per row
            for (; unit < n_units && tile == cur_tile; ) {
                const int sc = unit / S, ph = unit - sc * S;
                const int chunk = 2 * sc + half;               // 32-channel chunk of this group (may not exist: odd n_chunks)
                const uint32_t par = aphase ^ 1;
                uint8_t* hi = smA + as * L.a_stage;
                uint8_t* lo = hi + L.a_rows * 128;
                const uint32_t c16 = (uint32_t)(half * 4 + (jchunk >> 1)), sub8 = (uint32_t)((jchunk & 1) << 3);
                if (p.dbg & 512) {
                    wait_a_empty(a_empty + as, par);
                } else if (chunk >= n_chunks) {
                    wait_a_empty(a_empty + as, par);      // missing half of the last stage: never read by the MMAs
                } else if (PAIR || raw) {
                    // ---- TMA-staged unit: the dense [a_rows][32 ch] boxes (+ the coefficient slices) wait in the raw ring; rows go
                    // shared -> registers -> shared one at a time (no long-latency loads to batch, few live registers)
                    bool c_ok = chunk * TC_KC + jchunk * 4 < C_in;
                    if (FREQ && p.pad_zero) {              // a zero-padded frequency tap contributes nothing (its box arrives zero-filled)
                        const int f_src = f_out * p.fq.SF + (chunk * TC_KC) / pitch - p.fq.pad_f;
                        c_ok = c_ok && f_src >= 0 && f_src < p.fq.F_in;
                    }
                    const int idx = 2 * S * sc + ((2 * sc + 1 < n_chunks) ? 2 * ph + half : ph);
                    const int rc = rawbase + idx;
                    const int rslot = rc % nraw;
                    mbar_wait(raw_full + rslot, (uint32_t)((rc / nraw) & 1));
                    const uint8_t* rb = smR + rslot * L.raw_slot;
                    float4 a0 = make_float4(in_scale, in_scale, in_scale, in_scale), b0 = make_float4(0.f, 0.f, 0.f, 0.f), a1 = a0, b1 = b0;
                    if (!c_ok) { a0 = b0; a1 = b0; }
                    else {
                        if (cf0) {
                            a0 = *reinterpret_cast<const float4*>(rb + L.raw_cf + jchunk * 16); b0 = *reinterpret_cast<const float4*>(rb + L.raw_cf + 128 + jchunk * 16);
                            a0.x *= in_scale; a0.y *= in_scale; a0.z *= in_scale; a0.w *= in_scale;
                            b0.x *= in_scale; b0.y *= in_scale; b0.z *= in_scale; b0.w *= in_scale;
                        }
                        if (cf1) {
                            a1 = *reinterpret_cast<const float4*>(rb + L.raw_cf + 256 + jchunk * 16); b1 = *reinterpret_cast<const float4*>(rb + L.raw_cf + 384 + jchunk * 16);
                            a1.x *= in_scale; a1.y *= in_scale; a1.z *= in_scale; a1.w *= in_scale;
                            b1.x *= in_scale; b1.y *= in_scale; b1.z *= in_scale; b1.w *= in_scale;
                        }
                    }
                    wait_a_empty(a_empty + as, par);
                    const uint8_t* rrow = rb + rsub * raw_pitch + jchunk * 16;
                    // edge tiles apply the index map per row; interior tiles compile without it
                    auto raw_rows = [&](auto edge_c) {
                        constexpr bool EDGE = decltype(edge_c)::value;
                        constexpr int UNROLL = EDGE ? 1 : NR;  // the edge body, unrolled, does not fit the producer register budget
#pragma unroll UNROLL
                        for (int i = 0; i < NR_RAW; ++i) {
                            const int u = r0 + rsub + TC_PROWS * i;
                            if (u < r_end) {
                                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                                bool ok = c_ok, from_gl = false;
                                long long goff = 0;
                                if (EDGE) {
                                    // the index map of the per-thread path: a zero row stays zero; a reflected row, or one the tensor map
                                    // does not cover, is read from global memory; every other row is the box row
                                    const int gt = (t0 + u) * S + ph - p.pad_l;
                                    int src = gt;
                                    ok = ok && gt <= gt_max;
                                    if (p.pad_zero) ok = ok && gt >= 0 && gt < p.T_in;
                                    else { src = reflect_index(gt, p.T_ext); ok = ok && src < p.T_in && src >= 0; }
                                    from_gl = src != gt || gt >= tq_rows * S;
                                    goff = (long long)src * C_in + chunk * TC_KC + jchunk * 4;
                                }
                                if (ok) {
                                    const float4 xv = from_gl ? __ldg(reinterpret_cast<const float4*>(x0 + goff))
                                                              : *reinterpret_cast<const float4*>(rrow + i * TC_PROWS * raw_pitch);
                                    v.x = fmaf(xv.x, a0.x, b0.x); v.y = fmaf(xv.y, a0.y, b0.y);
                                    v.z = fmaf(xv.z, a0.z, b0.z); v.w = fmaf(xv.w, a0.w, b0.w);
                                    if (has1) {
                                        const float4 yv = from_gl ? __ldg(reinterpret_cast<const float4*>(x1 + goff))
                                                                  : *reinterpret_cast<const float4*>(rrow + L.raw_in1 + i * TC_PROWS * raw_pitch);
                                        v.x = v.x + fmaf(yv.x, a1.x, b1.x); v.y = v.y + fmaf(yv.y, a1.y, b1.y);
                                        v.z = v.z + fmaf(yv.z, a1.z, b1.z); v.w = v.w + fmaf(yv.w, a1.w, b1.w);
                                    }
                                    if (p.elu) {
                                        v.x = elu_scaled(v.x, p.tc_elu_k, in_scale); v.y = elu_scaled(v.y, p.tc_elu_k, in_scale);
                                        v.z = elu_scaled(v.z, p.tc_elu_k, in_scale); v.w = elu_scaled(v.w, p.tc_elu_k, in_scale);
                                    }
                                }
                                if (p.dbg & 4) continue;
                                uint2 h, l;
                                split_f16x2(v.x, v.y, h.x, l.x);
                                split_f16x2(v.z, v.w, h.y, l.y);
                                const uint32_t o = (uint32_t)u * 128u + ((c16 ^ (uint32_t)(u & 7)) << 4) + sub8;
                                *reinterpret_cast<uint2*>(hi + o) = h;
                                *reinterpret_cast<uint2*>(lo + o) = l;
                            }
                        }
                    };
                    if (edge) raw_rows(std::true_type{}); else raw_rows(std::false_type{});
                    mbar_arrive(raw_empty + rslot);            // the raw rows have been consumed
                    fence_proxy_async_smem();
                } else {
                int c = chunk * TC_KC + jchunk * 4;
                bool c_ok = c < C_in;
                const float* xu0 = x0;
                const float* xu1 = x1;
                if (FREQ) {
                    // gathered channel -> (frequency tap, stored channel); the tap selects the input row of this thread
                    const int kf = c / pitch;
                    c -= kf * pitch;
                    int f_src = f_out * p.fq.SF + kf - p.fq.pad_f;
                    if (p.pad_zero) c_ok = c_ok && f_src >= 0 && f_src < p.fq.F_in;
                    else f_src = reflect_index(f_src, p.fq.F_in);
                    if (!c_ok) f_src = 0;
                    xu0 = x0 + (long long)(p.fq.f_off0 + f_src) * p.fq.T_raw0 * pitch;
                    if (has1) xu1 = x1 + (long long)(p.fq.f_off1 + f_src) * p.fq.T_raw1 * pitch;
                }
                // the operand scale (a power of two: exact) is folded into the deferred-GroupNorm affine
                float4 a0 = make_float4(in_scale, in_scale, in_scale, in_scale), b0 = make_float4(0.f, 0.f, 0.f, 0.f), a1 = a0, b1 = b0;
                if (!c_ok) { a0 = b0; a1 = b0; }
                else if (cf0) {
                    a0 = __ldg(reinterpret_cast<const float4*>(cf0 + c)); b0 = __ldg(reinterpret_cast<const float4*>(cf0 + pitch + c));
                    a0.x *= in_scale; a0.y *= in_scale; a0.z *= in_scale; a0.w *= in_scale;
                    b0.x *= in_scale; b0.y *= in_scale; b0.z *= in_scale; b0.w *= in_scale;
                }
                if (c_ok && cf1) {
                    a1 = __ldg(reinterpret_cast<const float4*>(cf1 + c)); b1 = __ldg(reinterpret_cast<const float4*>(cf1 + pitch + c));
                    a1.x *= in_scale; a1.y *= in_scale; a1.z *= in_scale; a1.w *= in_scale;
                    b1.x *= in_scale; b1.y *= in_scale; b1.z *= in_scale; b1.w *= in_scale;
                }
                // row loads go out PB passes at a time (what the producer register budget holds); the first batch is issued
                // before the ring slot is waited for
                constexpr int PB = 3;
                static_assert(NR % PB == 0, "whole batches");
#pragma unroll
                for (int i0 = 0; i0 < NR; i0 += PB) {
                    float4 xa[PB], xb[PB];
                    bool okr[PB];
#pragma unroll
                    for (int j = 0; j < PB; ++j) {
                        const int u = rsub + TC_PROWS * (i0 + j);
                        const int gt = (t0 + u) * S + ph - p.pad_l;
                        bool ok = c_ok && u < L.a_rows && gt <= gt_max;
                        int src = gt;
                        if (p.pad_zero) ok = ok && gt >= 0 && gt < p.T_in;
                        else { src = reflect_index(gt, p.T_ext); ok = ok && src < p.T_in && src >= 0; }
                        okr[j] = ok;
                        xa[j] = make_float4(0.f, 0.f, 0.f, 0.f);
                        xb[j] = xa[j];
                        if (ok && !(p.dbg & 1)) {
                            const long long off = (long long)src * pitch + c;
                            xa[j] = __ldg(reinterpret_cast<const float4*>(xu0 + off));
                            if (has1) xb[j] = __ldg(reinterpret_cast<const float4*>(xu1 + off));
                        }
                    }
                    if (i0 == 0) {
                        wait_a_empty(a_empty + as, par);
                    }
#pragma unroll
                    for (int j = 0; j < PB; ++j) {
                        const int u = rsub + TC_PROWS * (i0 + j);
                        if (u < L.a_rows) {
                            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                            if (p.dbg & 2) v = xa[j];
                            else if (okr[j]) {
                                const float4 xv = xa[j];
                                v.x = fmaf(xv.x, a0.x, b0.x); v.y = fmaf(xv.y, a0.y, b0.y);
                                v.z = fmaf(xv.z, a0.z, b0.z); v.w = fmaf(xv.w, a0.w, b0.w);
                                if (has1) {
                                    const float4 yv = xb[j];
                                    v.x = v.x + fmaf(yv.x, a1.x, b1.x); v.y = v.y + fmaf(yv.y, a1.y, b1.y);
                                    v.z = v.z + fmaf(yv.z, a1.z, b1.z); v.w = v.w + fmaf(yv.w, a1.w, b1.w);
                                }
                                if (p.elu) {
                                    v.x = elu_scaled(v.x, p.tc_elu_k, in_scale); v.y = elu_scaled(v.y, p.tc_elu_k, in_scale);
                                    v.z = elu_scaled(v.z, p.tc_elu_k, in_scale); v.w = elu_scaled(v.w, p.tc_elu_k, in_scale);
                                }
                            }
                            if (p.dbg & 4) continue;
                            uint2 h, l;
                            split_f16x2(v.x, v.y, h.x, l.x);
                            split_f16x2(v.z, v.w, h.y, l.y);
                            const uint32_t o = (uint32_t)u * 128u + ((c16 ^ (uint32_t)(u & 7)) << 4) + sub8;
                            *reinterpret_cast<uint2*>(hi + o) = h;
                            *reinterpret_cast<uint2*>(lo + o) = l;
                        }
                    }
                }
                fence_proxy_async_smem();
                }
                mbar_arrive(a_full + as);
                if (R::PROD_GROUPS == 1 && split && half == 0) { half = 1; continue; }   // the stage's second half
                if (PAIR) {
                    // every producer thread has fenced its stores to the async proxy; one thread then copies the rows to the peer
                    // and posts, with the one extra local arrival, the bytes the peer copies into this stage (a peer copy that
                    // completes first only drives the tx-count below zero: the pending arrival keeps the phase open).  The source
                    // rows are not overwritten before the copy has read them: the next write of this stage waits for a_empty,
                    // which the peer's consumers arrive on only after the peer's a_full -- and so this copy -- has completed.
                    asm volatile("bar.sync 2, 128;" ::: "memory");
                    if (ptid == 0) {
                        const uint32_t so = (uint32_t)(as * L.a_stage + r0 * 128);
                        bulk_s2peer(smA_peer + so, smA + so, hand_bytes, a_full_peer + 8u * (uint32_t)as);
                        bulk_s2peer(smA_peer + so + L.a_rows * 128, smA + so + L.a_rows * 128, hand_bytes, a_full_peer + 8u * (uint32_t)as);
                        mbar_arrive_expect_tx(a_full + as, peer_bytes);
                    }
                }
                half = half0;
                as += step;
                if (as >= na_stages) { as -= na_stages; aphase ^= 1; }
                unit += step;
            }
            while (unit >= n_units && tile < n_tiles) {
                if (tile_raw(tc_tile(tile, n_nt, n_tt).tt * TC_M)) rawbase += units_per_tile;
                unit -= n_units; tile += gridDim.x;
            }
        }
    } else if (role == R::CTL_WG) {
        // =========================================================== control warpgroup: weight slabs (its warp 0), raw tiles (warp 1)
        setmaxnreg_dec<R::CTL_REGS>();
        if (warp == 4 * R::CTL_WG && lane == 0) {
            // weight slabs via the bulk-copy engine
            const uint32_t bytes = (uint32_t)L.b_stage;
            int bs = 0;
            uint32_t bphase = 0;
            bool first = true;
            for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
                if (w_resident && !first) break;                       // whole layer image already resident
                const TcTile tl = tc_tile(tile, n_nt, n_tt);
                const uint8_t* wbase = reinterpret_cast<const uint8_t*>(p.w_tc) + (long long)tl.nt * n_sc * K * bytes;
                int chunk = 0, ph = 0;                                 // chunk: 64-channel stage chunk
                for (int unit = 0; unit < n_units; ++unit) {
                    for (int k = ph; k < K; k += S) {
                        if (!w_resident) { if (p.dbg & 64) mbar_wait(b_empty + bs, bphase ^ 1); else mbar_wait_backoff(b_empty + bs, bphase ^ 1, 64); }
                        if (p.dbg & 256) { mbar_arrive(b_full + bs); }
                        else {
                            mbar_arrive_expect_tx(b_full + bs, bytes);
                            bulk_g2s(smB + bs * L.b_stage, wbase + ((long long)chunk * K + k) * bytes, bytes, b_full + bs);
                        }
                        if (++bs == nb_stages) { bs = 0; bphase ^= 1; }
                    }
                    if (++ph == S) { ph = 0; ++chunk; }
                }
                first = false;
            }
        } else if (warp == 4 * R::CTL_WG + 1 && lane == 0 && nraw > 0 && !(p.dbg & 512)) {
            // raw activation tiles via TMA (cp.async.bulk.tensor)
            const uint32_t row_bytes = (uint32_t)(ka.raw_rows * raw_pitch);   // the box: this CTA's share of the slab rows
            const uint32_t cbytes = (uint32_t)raw_pitch;
            const uint32_t n_cf = (p.in0.coef ? 2u : 0u) + ((has1 && p.in1.coef) ? 2u : 0u);
            const uint32_t unit_bytes = row_bytes * (has1 ? 2u : 1u) + n_cf * cbytes;
            int rc = 0;
            for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
                const TcTile tl = tc_tile(tile, n_nt, n_tt);
                const int t0 = tl.tt * TC_M;
                if (!tile_raw(t0)) continue;
                int b = tl.b, f_out = 0;
                if (FREQ) { b = tl.b / p.fq.F_out; f_out = tl.b - b * p.fq.F_out; }
                const int pitch = FREQ ? p.fq.cin : C_in;
                const float* cf0 = p.in0.coef ? p.in0.coef + (long long)b * 2 * pitch : nullptr;
                const float* cf1 = (has1 && p.in1.coef) ? p.in1.coef + (long long)b * 2 * pitch : nullptr;
                for (int sc = 0; sc < n_sc; ++sc)
                    for (int ph = 0; ph < S; ++ph) {
                        // row (t0 + u) * S + ph - pad_l == (tq0 + u) * S + php
                        const int r = ph - p.pad_l;
                        const int fd = (r >= 0) ? r / S : -((-r + S - 1) / S);
                        const int tq0 = t0 + fd, php = r - fd * S;
                        for (int hh = 0; hh < 2; ++hh) {
                            const int chunk = 2 * sc + hh;
                            if (chunk >= n_chunks) break;
                            const int slot = rc % nraw;
                            mbar_wait(raw_empty + slot, (uint32_t)((rc / nraw) & 1) ^ 1);
                            uint8_t* dst = smR + slot * L.raw_slot;
                            mbar_arrive_expect_tx(raw_full + slot, unit_bytes);
                            int c0 = chunk * TC_KC;            // first stored channel of the unit
                            if (FREQ) {
                                // gathered chunk -> (frequency tap, 32-channel slice of it); a reflected tap is just another row,
                                // a zero-padded one is out of bounds for the tensor map (zero fill)
                                const int kf = c0 / pitch;
                                c0 -= kf * pitch;
                                int f_src = f_out * p.fq.SF + kf - p.fq.pad_f;
                                if (!p.pad_zero) f_src = reflect_index(f_src, p.fq.F_in);
                                tma_load_5d(dst, &tm0, c0, php, tq0, f_src, b, raw_full + slot);
                                if (has1) tma_load_5d(dst + L.raw_in1, &tm1, c0, php, tq0, f_src, b, raw_full + slot);
                            } else {
                                tma_load_4d(dst, &tm0, c0, php, tq0 + r0, b, raw_full + slot);
                                if (has1) tma_load_4d(dst + L.raw_in1, &tm1, c0, php, tq0 + r0, b, raw_full + slot);
                            }
                            if (cf0) {
                                bulk_g2s(dst + L.raw_cf, cf0 + c0, cbytes, raw_full + slot);
                                bulk_g2s(dst + L.raw_cf + 128, cf0 + pitch + c0, cbytes, raw_full + slot);
                            }
                            if (cf1) {
                                bulk_g2s(dst + L.raw_cf + 256, cf1 + c0, cbytes, raw_full + slot);
                                bulk_g2s(dst + L.raw_cf + 384, cf1 + pitch + c0, cbytes, raw_full + slot);
                            }
                            ++rc;
                        }
                    }
            }
        }
    } else {
        // =========================================================== consumer warpgroups: wgmma issue, group fold, epilogue
        setmaxnreg_inc<R::CONS_REGS>();
        constexpr int NA = N_TILE / 2;                            // accumulator registers per thread (m64 x N_TILE per warpgroup)
        constexpr int PARTS = R::PARTS;
        const int cw = warp - 4 * R::CONS_WG;                     // 0..7
        const int wg = cw >> 2;                                   // tile rows 64*wg .. 64*wg + 63
        const int ctid = tid - 128 * R::CONS_WG;                  // 0..255
        const bool leader = (tid & 127) == 0;                     // one arrival per warpgroup on the ring barriers
        const uint32_t a_base = smem_u32(smA) + (uint32_t)(wg * 64 * 128), b_base = smem_u32(smB);
        const uint32_t a_empty_peer = PAIR ? mapa_shared(smem_u32(a_empty), peer) : 0u;   // PAIR: the peer wrote rows of our stages
        const int r_lo = wg * 64 + (cw & 3) * 16 + (lane >> 2);   // accumulator rows of this thread: r_lo, r_lo + 8
        const int cq = 2 * (lane & 3);                            // first of its two columns in every 8-column group
        // 2-D plain convs (no phase scatter, no padded columns) store [pseudo-clip][t][C_out] like a 1-D layer
        const bool plain_out = FREQ && p.fq.FR == 1 && p.fq.TR == 1 && p.fq.c_store == p.C_out;
        const float out_scale = p.tc_out_scale;
        // fused GroupNorm finalisation: partials of the current clip written by this CTA since the last report
        int fin_clip = -1, fin_local = 0;
        auto fin_flush = [&]() {
            // all 256 consumer threads call this together.  Report this CTA's partial count for fin_clip; whoever completes the
            // clip reduces ALL its partials in a fixed order (independent of which CTA does it) and writes stats + affine.
            if (fin_clip < 0 || fin_local == 0) return;
            int* flag = reinterpret_cast<int*>(red + 16 * PARTS);
            if (ctid == 0) {
                __threadfence();                                         // this CTA's partials before the count
                const int old = atomicAdd(p.fin_counter + fin_clip, fin_local);
                *flag = (old + fin_local == p.fin_parts) ? 1 : 0;
            }
            asm volatile("bar.sync 1, 256;" ::: "memory");
            const bool last_cta = *flag != 0;
            if (last_cta) {
                __threadfence();                                         // the other CTAs' partials after the count
                const double* pp = p.partials + (long long)fin_clip * p.fin_parts * 2;
                double fs = 0.0, fss = 0.0;
                for (int i = ctid; i < p.fin_parts; i += 256) { fs += __ldcg(pp + 2 * i); fss += __ldcg(pp + 2 * i + 1); }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) {
                    fs += __shfl_xor_sync(0xffffffffu, fs, o);
                    fss += __shfl_xor_sync(0xffffffffu, fss, o);
                }
                asm volatile("bar.sync 1, 256;" ::: "memory");          // everyone has read the flag
                if (lane == 0) { red[cw * 2] = fs; red[cw * 2 + 1] = fss; }
                asm volatile("bar.sync 1, 256;" ::: "memory");
                double ts = 0.0, tss = 0.0;
#pragma unroll
                for (int w = 0; w < 8; ++w) { ts += red[2 * w]; tss += red[2 * w + 1]; }
                const double mean_d = ts / p.fin_count;
                double var = tss / p.fin_count - mean_d * mean_d;
                if (var < 0.0) var = 0.0;
                const float mean = (float)mean_d, rstd = (float)(1.0 / sqrt(var + (double)p.fin_eps));
                if (ctid == 0) {
                    p.fin_stats[2 * fin_clip] = mean;
                    p.fin_stats[2 * fin_clip + 1] = rstd;
                    p.fin_counter[fin_clip] = 0;                         // ready for the next launch
                }
                if (p.fin_coef)
                    for (int c = ctid; c < p.fin_C; c += 256) {
                        const float a = rstd * p.fin_gamma[c];
                        p.fin_coef[(long long)fin_clip * 2 * p.fin_C + c] = a;
                        p.fin_coef[(long long)fin_clip * 2 * p.fin_C + p.fin_C + c] = p.fin_beta[c] - a * mean;
                    }
            }
            asm volatile("bar.sync 1, 256;" ::: "memory");              // `red` / flag free again
            fin_local = 0;
        };
        int as = 0, bs = 0;
        uint32_t aphase = 0, bphase = 0;
        bool first = true;
        float acc[NA], tot[NA];
        for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
            const TcTile tl = tc_tile(tile, n_nt, n_tt);
            int ph = 0;
            if (w_resident) bs = 0;
            // a ring stage is released once the wgmma that read it have completed: one commit group per tap, at most one
            // group in flight behind the one just issued
            int pend_a = -1, pend_b = -1;
            for (int g = 0; g < n_groups; ++g) {
                uint32_t accum = 0;
                const int u_end = min(n_units, (g + 1) * upg);
                for (int unit = g * upg; unit < u_end; ++unit) {
                    mbar_wait(a_full + as, aphase);
                    const uint32_t a_hi0 = a_base + as * L.a_stage;
                    const uint32_t a_lo0 = a_hi0 + L.a_rows * 128;
                    // K steps of 16 channels: 4 for a full 64-channel stage, 2 when only its first half exists
                    const bool full_stage = 2 * (unit / S) + 1 < n_chunks;
                    int q = 0;
                    for (int k = ph; k < K; k += S, ++q) {
                        if (!w_resident || first) mbar_wait(b_full + bs, bphase);
                        const uint32_t b_hi0 = b_base + bs * L.b_stage;
                        const uint32_t b_lo0 = b_hi0 + N_TILE * 128;
                        if (full_stage) tc_issue_tap<N_TILE, 4>(acc, a_hi0 + q * 128, a_lo0 + q * 128, b_hi0, b_lo0, accum);
                        else tc_issue_tap<N_TILE, 2>(acc, a_hi0 + q * 128, a_lo0 + q * 128, b_hi0, b_lo0, accum);
                        accum = 1;
                        wgmma_wait<1>();
                        // the previous tap's commit group has completed: release what only it read (predicated, no branch)
                        mbar_arrive_if(b_empty + pend_b, leader && pend_b >= 0);
                        mbar_arrive_if(a_empty + pend_a, leader && pend_a >= 0);
                        if (PAIR) mbar_arrive_remote_if(a_empty_peer + 8u * (uint32_t)pend_a, leader && pend_a >= 0);
                        pend_b = w_resident ? -1 : bs;
                        pend_a = -1;
                        if (++bs == nb_stages) { bs = 0; bphase ^= 1; }
                    }
                    pend_a = as;
                    if (++as == na_stages) { as = 0; aphase ^= 1; }
                    if (++ph == S) ph = 0;
                }
                wgmma_wait<0>();
                reg_fence(acc);
                if (leader) {
                    if (pend_b >= 0) mbar_arrive(b_empty + pend_b);
                    if (pend_a >= 0) mbar_arrive(a_empty + pend_a);
                    if (PAIR && pend_a >= 0) mbar_arrive_remote_if(a_empty_peer + 8u * (uint32_t)pend_a, true);
                }
                pend_a = -1; pend_b = -1;
#pragma unroll
                for (int i = 0; i < NA; ++i) tot[i] = g == 0 ? acc[i] : tot[i] + acc[i];
            }
            first = false;
            // ---- epilogue: bias, raw store, GroupNorm partial statistics
            long long frow = 0;                                       // FREQ: element row of (clip, f_out*FR, t = 0)
            if (FREQ) {
                const int fb = tl.b / p.fq.F_out, ff = tl.b - fb * p.fq.F_out;
                frow = ((long long)fb * p.fq.F_out * p.fq.FR + (long long)ff * p.fq.FR) * ((long long)p.T_out * p.fq.TR);
            }
            const float* bias = p.bias + tl.nt * N_TILE;
            float s[PARTS], ss[PARTS];                                // per 64-column part of the tile
#pragma unroll
            for (int hp = 0; hp < PARTS; ++hp) { s[hp] = 0.f; ss[hp] = 0.f; }
#pragma unroll
            for (int j = 0; j < N_TILE / 8; ++j) {
                const int c = 8 * j + cq;
                const int hp = j * PARTS / (N_TILE / 8);
                const float bias0 = __ldg(bias + c), bias1 = __ldg(bias + c + 1);
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int t = tl.tt * TC_M + r_lo + 8 * h;
                    if (t >= p.T_out) continue;
                    // exact power-of-two rescale + bias in one rounding (== fl(acc / scale + bias))
                    float2 o;
                    o.x = fmaf(tot[4 * j + 2 * h], out_scale, bias0);
                    o.y = fmaf(tot[4 * j + 2 * h + 1], out_scale, bias1);
                    s[hp] += o.x + o.y;
                    ss[hp] = fmaf(o.x, o.x, ss[hp]); ss[hp] = fmaf(o.y, o.y, ss[hp]);
                    if (p.dbg & 8) continue;
                    if (!FREQ || plain_out) {
                        *reinterpret_cast<float2*>(p.out + (long long)tl.b * p.out_clip_stride + (long long)t * p.C_out + tl.nt * N_TILE + c) = o;
                    } else {
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            // phase (pf, pt) of a transposed conv lands on row f_out*FR + pf, column t*TR + pt; padded columns of
                            // the n-tile (channel >= c_store) do not exist in HBM
                            const int co = tl.nt * N_TILE + c + e;
                            const int phs = co / p.fq.Cc, cch = co - phs * p.fq.Cc;
                            if (cch < p.fq.c_store) {
                                const int pf = phs / p.fq.TR, pt = phs - pf * p.fq.TR;
                                p.out[(frow + (long long)t * p.fq.TR + (long long)pf * p.T_out * p.fq.TR + pt) * p.fq.c_store + cch] = e ? o.y : o.x;
                            }
                        }
                    }
                }
            }
            if (p.partials && !(p.dbg & 16)) {
                // one partial per 64-column part, at the index a 64-column tile of those columns has: the layer's partials and
                // their reduction order are the same whatever the tile width
                double ds[PARTS], dss[PARTS];
#pragma unroll
                for (int hp = 0; hp < PARTS; ++hp) {
                    ds[hp] = (double)s[hp]; dss[hp] = (double)ss[hp];
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) {
                        ds[hp] += __shfl_xor_sync(0xffffffffu, ds[hp], o);
                        dss[hp] += __shfl_xor_sync(0xffffffffu, dss[hp], o);
                    }
                }
                asm volatile("bar.sync 1, 256;" ::: "memory");      // previous tile's reader is done with `red`
                if (lane == 0) {
#pragma unroll
                    for (int hp = 0; hp < PARTS; ++hp) { red[(hp * 8 + cw) * 2] = ds[hp]; red[(hp * 8 + cw) * 2 + 1] = dss[hp]; }
                }
                asm volatile("bar.sync 1, 256;" ::: "memory");
                if (ctid < PARTS) {
                    const int hp = ctid;
                    const int nparts = n_nt * PARTS * n_tt;
                    double* dst = p.partials + ((long long)tl.b * nparts + (tl.nt * PARTS + hp) * n_tt + tl.tt) * 2;
                    double ts = 0.0, tss = 0.0;
#pragma unroll
                    for (int w = 0; w < 8; ++w) { ts += red[(hp * 8 + w) * 2]; tss += red[(hp * 8 + w) * 2 + 1]; }
                    dst[0] = ts;
                    dst[1] = tss;
                }
                if (p.fin_counter) {
                    const int clip = FREQ ? tl.b / p.fq.F_out : tl.b;
                    if (clip != fin_clip) { fin_flush(); fin_clip = clip; }
                    fin_local += PARTS;
                }
            }
        }
        if (p.fin_counter && p.partials && !(p.dbg & 16)) fin_flush();
    }
    // PAIR: no CTA exits while its peer can still copy into its shared memory or arrive on its barriers
    if (PAIR) cluster_sync();
#undef na_stages
#undef nb_stages
#undef n_tiles
#undef w_resident
#undef nraw
#undef raw_pitch
#undef n_chunks
#undef n_sc
#undef n_units
#undef upg
#undef n_groups
#undef n_tt
#undef n_nt
#undef units_per_tile
#undef tq_rows
}

// ------------------------------------------------------------------------------------------ host side
bool conv_tc_supported(int C_in, int C_out_eff, int K, int S, int D) {
    return D == 1 && (C_in % TC_KC == 0 || C_in == 16) && C_out_eff % 16 == 0 && K >= 1 && S >= 1 && ((K - 1) / S) <= 16;
}

// 2-D mode: cin stored channels per input element, C_out_eff output columns of the (possibly n-tile padded) weight image
bool conv_tc_supported_2d(int cin, int C_out_eff, int KT, int ST) {
    const bool cin_ok = cin % 4 == 0 && (cin % TC_KC == 0 || TC_KC % cin == 0);   // a thread's 4 channels share one tap
    return cin_ok && C_out_eff % 16 == 0 && KT >= 1 && ST >= 1 && ((KT - 1) / ST) <= 16;
}

// output columns per GroupNorm partial (and per tile up to 64)
static int tc_part_cols(int C_out_eff) {
    if (C_out_eff % 64 == 0) return 64;
    if (C_out_eff % 32 == 0) return 32;
    return 16;
}

// Output columns per tile.  1-D layers with C_out_eff % 128 == 0 take 128-column tiles (the 4-warpgroup layout of TcRoles), so
// each activation element is transformed once per 128 columns; the 2-D mode stays at <= 64.  The weight packer and the launcher
// both take the tile width from here.
int conv_tc_n_tile(int C_out_eff, bool freq) {
    if (!freq && C_out_eff % 128 == 0) return 128;
    return tc_part_cols(C_out_eff);
}

int conv_tc_num_parts(int T_out, int C_out_eff) {
    return ((T_out + TC_M - 1) / TC_M) * (C_out_eff / tc_part_cols(C_out_eff));
}

static int g_num_sms = 0;

static int g_group_mmas = TC_GROUP_MMAS, g_deep_ring = 1, g_dbg = 0, g_na_tma = 2;

struct TcPlan { int resident, na, nb, nraw; TcSmemLayout L; bool ok; };

// shared-memory plan: weights resident (small layers: the whole image of the single n-tile) or streamed through a ring as
// deep as fits; A ring `na_first` stages (4, else 2) -- with a raw TMA ring the A ring only decouples producers from the MMA
// issue, so 2 stages suffice and the rest of the shared memory buys prefetch depth (nraw units in flight).
// At N_TILE = 128 a B stage is 32 KB; the last fallback (na = nb = 2) still fits every supported shape: A 2 x 36 KB (144 rows)
// + B 2 x 32 KB + two raw slots of a two-input unit (2 x 36.5 KB) + barriers and scratch = 209.5 KB of 225.
// pair: the raw slots hold a 2-CTA pair's share of the slab rows (tc_layout), so they are half as large.  A pair asks for 3 A stages
// first: the copy to the peer and the release by both CTAs' consumers lengthen a stage's round trip, and with 2 stages the 1-tap
// layers lose more to that than they gain from the halved transform.  A pair whose stages feed two taps (the 8/4, 10/5 and 16/8 down
// convs, the up convs) asks for 2 B stages first, which leaves room for a deeper raw ring; with more taps per stage the B ring stays
// deeper (the k7 `dec.conv0` was 16 % slower at 2 B stages).  What the fallbacks below give, per (taps per stage, inputs):
//   1 tap,  one input:  na 3, nb 3, nraw 3      1 tap,  two inputs:  na 2, nb 3, nraw 3  (na 3 leaves no room for two raw slots)
//   2 taps, one input:  na 3, nb 2, nraw 6      2 taps, two inputs:  na 3, nb 2, nraw 3
//   3+ taps, one input: na 3, nb 3, nraw 2      3+ taps, two inputs: na 2, nb 3, nraw 3
static TcPlan tc_plan(const ConvParams& p, int na_first, bool want_raw, int g_deep_ring, bool pair = false) {
    const int limit = 225 * 1024;
    const int n_slabs = ((p.C_in + 2 * TC_KC - 1) / (2 * TC_KC)) * p.K;   // (64-channel stage chunk, tap) weight slabs per n-tile
    const int has1 = p.in1.x ? 1 : 0;
    const int cin_row = p.fq.KF > 0 ? p.fq.cin : p.C_in;                   // channels of a stored input row
    const int raw_pitch = (cin_row < TC_KC ? cin_row : TC_KC) * 4;
    TcPlan pl{};
    pl.ok = false;
    int na = pair ? 3 : na_first, nb = (pair && (p.K + p.S - 1) / p.S == 2) ? 2 : 4;
    TcSmemLayout L = tc_layout(p.K, p.S, p.n_tile, na, n_slabs);
    const int min_raw = want_raw ? 2 : 0;
    auto fits = [&](const TcSmemLayout& l) { return l.total + min_raw * tc_layout(p.K, p.S, p.n_tile, 2, 2, 1, raw_pitch, has1, pair).raw_slot <= limit; };
    if (n_slabs <= 64 && p.C_out == p.n_tile && fits(L)) { pl.resident = 1; nb = n_slabs; }   // one n-tile only
    else {
        L = tc_layout(p.K, p.S, p.n_tile, na, nb);
        if (!fits(L)) { nb = 3; L = tc_layout(p.K, p.S, p.n_tile, na, nb); }
        if (!fits(L)) { na = 2; nb = 4; L = tc_layout(p.K, p.S, p.n_tile, na, nb); }
        if (!fits(L)) { nb = 3; L = tc_layout(p.K, p.S, p.n_tile, na, nb); }
        if (!fits(L)) { nb = 2; L = tc_layout(p.K, p.S, p.n_tile, na, nb); }
        if (!fits(L)) return pl;
        // small n-tiles: a weight slab is only n_tile*256 bytes, so the ring is deepened until shared memory is full
        if (g_deep_ring && !want_raw)
            while (nb < 24 && nb < n_slabs && tc_layout(p.K, p.S, p.n_tile, na, nb + 1).total <= limit)
                L = tc_layout(p.K, p.S, p.n_tile, na, ++nb);
    }
    int nraw = 0;
    if (want_raw) {
        nraw = 2;
        while (nraw < TC_RAW_MAX && tc_layout(p.K, p.S, p.n_tile, na, nb, nraw + 1, raw_pitch, has1, pair).total <= limit) ++nraw;
    }
    pl.L = tc_layout(p.K, p.S, p.n_tile, na, nb, nraw, raw_pitch, has1, pair);
    pl.na = na; pl.nb = nb; pl.nraw = nraw;
    pl.ok = pl.L.total <= limit;
    return pl;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn g_encode_tiled = nullptr;
static int g_tma_state = 0;      // 0: not probed, 1: available, -1: unavailable / disabled (FCB_TC_TMA=0)

// 4-D view of a channels-last activation [B][T][C] that makes every stride phase a dimension: (channel, phase, row / S, clip).
// A unit of a tile = box {32 channels, 1 phase, a_rows rows, 1 clip}; rows beyond T / S (and before 0) are zero-filled.
static bool make_act_map(CUtensorMap* tm, const InView& v, int C, int S, int T_in, int B, int a_rows) {
    const float* base = v.x + (long long)v.row_off * C;
    const cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)S, (cuuint64_t)(T_in / S), (cuuint64_t)B};
    const cuuint64_t strides[3] = {(cuuint64_t)C * 4, (cuuint64_t)S * C * 4, (cuuint64_t)v.clip_stride * 4};
    const cuuint32_t box[4] = {(cuuint32_t)(C < TC_KC ? C : TC_KC), 1, (cuuint32_t)a_rows, 1};
    const cuuint32_t estr[4] = {1, 1, 1, 1};
    if (((uintptr_t)base & 15) != 0 || (strides[0] & 15) || (strides[2] & 15) || dims[2] == 0) return false;
    return g_encode_tiled(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float*>(base), dims, strides, box, estr,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// 2-D (FreqCodec) activation [B][F_raw][T_raw][cin]: (channel, phase, column / ST, frequency row, clip); the logical window
// starts at (f_off, t_off) and spans F_in x T_in -- taps outside it are out of bounds (zero fill) or reflected by the caller.
static bool make_act_map_2d(CUtensorMap* tm, const InView& v, int cin, int ST, int T_in, int F_in, int T_raw, int f_off, int B,
                            int a_rows) {
    const float* base = v.x + ((long long)f_off * T_raw + v.row_off) * cin;
    const cuuint64_t dims[5] = {(cuuint64_t)cin, (cuuint64_t)ST, (cuuint64_t)(T_in / ST), (cuuint64_t)F_in, (cuuint64_t)B};
    const cuuint64_t strides[4] = {(cuuint64_t)cin * 4, (cuuint64_t)ST * cin * 4, (cuuint64_t)T_raw * cin * 4,
                                   (cuuint64_t)v.clip_stride * 4};
    const cuuint32_t box[5] = {(cuuint32_t)(cin < TC_KC ? cin : TC_KC), 1, (cuuint32_t)a_rows, 1, 1};
    const cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    if (((uintptr_t)base & 15) != 0 || (strides[0] & 15) || (strides[2] & 15) || (strides[3] & 15) || dims[2] == 0) return false;
    return g_encode_tiled(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 5, const_cast<float*>(base), dims, strides, box, estr,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// 2-CTA clusters of the PAIR kernel a device holds at once (at 225 KB of shared memory each), per device ordinal: a process may
// drive devices of different models (ordinals beyond the table are queried at every launch)
constexpr int TC_PAIR_DEVICES = 64;
static int g_max_pairs[TC_PAIR_DEVICES] = {};

template <int N_TILE, bool FREQ, bool PAIR = false>
static cudaError_t launch_tc_n(const ConvParams& p, cudaStream_t st, const TcPlan& pl, int n_tiles, const CUtensorMap& tm0,
                               const CUtensorMap& tm1) {
    auto kern = conv1d_tc_kernel<N_TILE, FREQ, PAIR>;
    {
        cudaError_t e = ensure_dynamic_smem((const void*)kern, 225 * 1024);
        if (e != cudaSuccess) return e;
    }
    const int grid = n_tiles < g_num_sms ? n_tiles : g_num_sms;
    TcArgs ka{};
    ka.L = pl.L; ka.na = pl.na; ka.nb = pl.nb; ka.n_tiles = n_tiles; ka.w_resident = pl.resident; ka.nraw = pl.nraw;
    ka.n_chunks = (p.C_in + TC_KC - 1) / TC_KC;
    ka.n_sc = (ka.n_chunks + 1) >> 1;
    ka.split = ka.n_chunks > 1;
    ka.n_units = ka.n_sc * p.S;
    ka.upg = tc_units_per_group(p.K, p.S, g_group_mmas);
    ka.n_groups = (ka.n_units + ka.upg - 1) / ka.upg;
    ka.n_tt = (p.T_out + TC_M - 1) / TC_M;
    ka.n_nt = p.C_out / N_TILE;
    ka.units_per_tile = ka.n_chunks * p.S;
    ka.tq_rows = p.T_in / p.S;
    ka.raw_pitch = ((FREQ ? p.fq.cin : p.C_in) < TC_KC ? (FREQ ? p.fq.cin : p.C_in) : TC_KC) * 4;
    ka.raw_rows = tc_raw_rows(pl.L.a_rows, PAIR);
    if (PAIR) {
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeClusterDimension;
        attr[0].val.clusterDim.x = 2; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
        cudaLaunchConfig_t cfg = {};
        cfg.blockDim = dim3(TcRoles<N_TILE>::THREADS);
        cfg.stream = st;
        cfg.attrs = attr;
        cfg.numAttrs = 1;
        int dev = 0;
        cudaError_t e = cudaGetDevice(&dev);
        if (e != cudaSuccess) return e;
        int max_pairs = dev < TC_PAIR_DEVICES ? g_max_pairs[dev] : 0;
        if (max_pairs == 0) {
            int sms = 0;
            e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
            if (e != cudaSuccess) return e;
            cfg.gridDim = dim3(sms / 2 * 2);
            cfg.dynamicSmemBytes = 225 * 1024;
            e = cudaOccupancyMaxActiveClusters(&max_pairs, kern, &cfg);
            if (e != cudaSuccess) return e;
            if (max_pairs < 1) return cudaErrorInvalidConfiguration;
            if (dev < TC_PAIR_DEVICES) g_max_pairs[dev] = max_pairs;
        }
        // n_tiles is even (an even number of n-tiles per time tile), so both CTAs of a cluster walk the same number of tiles
        const int pairs = n_tiles / 2 < max_pairs ? n_tiles / 2 : max_pairs;
        cfg.gridDim = dim3(2 * pairs);
        cfg.dynamicSmemBytes = pl.L.total;
        return cudaLaunchKernelEx(&cfg, kern, p, ka, tm0, tm1);
    }
    kern<<<grid, TcRoles<N_TILE>::THREADS, pl.L.total, st>>>(p, ka, tm0, tm1);
    return cudaGetLastError();
}

template <int N_TILE>
static cudaError_t launch_tc_modes(const ConvParams& p, cudaStream_t st, const TcPlan& pl, int n_tiles, bool freq,
                                   const CUtensorMap& tm0, const CUtensorMap& tm1) {
    return freq ? launch_tc_n<N_TILE, true>(p, st, pl, n_tiles, tm0, tm1) : launch_tc_n<N_TILE, false>(p, st, pl, n_tiles, tm0, tm1);
}

cudaError_t launch_conv_tc(const ConvParams& p_in, int B, cudaStream_t st, int* nparts) {
    ConvParams p = p_in;
    if (g_num_sms == 0) {
        int dev = 0;
        cudaError_t e = cudaGetDevice(&dev);
        if (e != cudaSuccess) return e;
        e = cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
        if (e != cudaSuccess) return e;
        // tuning knobs (experiments only; defaults are the shipped configuration)
        if (const char* v = getenv("FCB_TC_GROUP_MMAS")) g_group_mmas = atoi(v) > 0 ? atoi(v) : TC_GROUP_MMAS;
        if (const char* v = getenv("FCB_TC_DEEP_RING")) g_deep_ring = atoi(v) != 0;
        if (const char* v = getenv("FCB_TC_DBG")) g_dbg = atoi(v);      // profiling knock-outs (wrong results)
        if (const char* v = getenv("FCB_TC_NA_TMA")) { const int f = atoi(v); if (f == 2 || f == 4) g_na_tma = f; }
        // TMA staging of the activation tiles: cuTensorMapEncodeTiled through the runtime's driver entry point (no -lcuda)
        g_tma_state = -1;
        const char* tv = getenv("FCB_TC_TMA");
        if (!tv || atoi(tv) != 0) {
            void* fn = nullptr;
            cudaDriverEntryPointQueryResult qres;
            if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) == cudaSuccess && fn &&
                qres == cudaDriverEntryPointSuccess) {
                g_encode_tiled = (EncodeTiledFn)fn;
                g_tma_state = 1;
            }
        }
    }
    p.dbg = g_dbg;
    if (!(p.tc_in_scale > 0.f)) p.tc_in_scale = 16.f;           // post-GroupNorm activations are O(1): 16 x keeps |x| < 4094 finite
    if (!(p.tc_w_scale > 0.f)) p.tc_w_scale = 1.f;
    p.tc_out_scale = 1.0f / (p.tc_in_scale * p.tc_w_scale);     // powers of two: exact
    p.tc_elu_k = 1.4426950408889634f / p.tc_in_scale;
    const int n_tt = (p.T_out + TC_M - 1) / TC_M, n_nt = p.C_out / p.n_tile;
    *nparts = n_tt * (p.C_out / tc_part_cols(p.C_out));
    const int n_tiles = n_tt * n_nt * B;
    const bool freq = p.fq.KF > 0;          // B counts pseudo-clips (clips x output frequency rows) in the 2-D mode
    // raw TMA ring: every 1-D layer (edge tiles included) and the 2-D layers with interior tiles, channel counts the box covers,
    // 16-byte aligned views
    CUtensorMap tm0{}, tm1{};
    // (2-D: a 32-channel unit must be a slice of ONE frequency tap -> cin % 32 == 0, or the single tap of a 16-channel 1x1 conv)
    // (2-D: interior tiles exist when the clip has at least 3 tiles, or for 1x1 layers -- no halo -- always)
    bool want_raw = g_tma_state == 1 && (!freq || n_tt >= 3 || (p.K == 1 && p.S == 1 && p.pad_l == 0)) && p.T_in / p.S >= 1 &&
                    (freq ? (p.fq.cin % TC_KC == 0 || (p.fq.cin == 16 && p.fq.KF == 1)) : (p.C_in % TC_KC == 0 || p.C_in == 16));
    // 2-D layers: built and parity-tested (5-D tensor maps) but opt-in (FCB_TC_TMA2D=1): the K_F-fold re-read of every input row
    // makes the unit stream L2-bound either way and the TMA path adds a hand-off
    if (freq && !(getenv("FCB_TC_TMA2D") && atoi(getenv("FCB_TC_TMA2D")) != 0)) want_raw = false;
    // 2-CTA pairs (conv1d_tc_kernel<128, false, true>): 1-D 128-column layers on the raw ring with an even number of n-tiles, whose
    // CTAs would otherwise each fetch and transform the same activation rows
    const bool pair = !freq && p.n_tile == 128 && n_nt % 2 == 0;
    TcPlan pl{};
    if (want_raw) {
        pl = tc_plan(p, g_na_tma, true, g_deep_ring, pair);
        want_raw = pl.ok && pl.nraw >= 2;
        if (want_raw && !freq)
            want_raw = make_act_map(&tm0, p.in0, p.C_in, p.S, p.T_in, B, tc_raw_rows(pl.L.a_rows, pair)) &&
                       (!p.in1.x || make_act_map(&tm1, p.in1, p.C_in, p.S, p.T_in, B, tc_raw_rows(pl.L.a_rows, pair)));
        if (want_raw && freq) {
            const int nclips = B / p.fq.F_out;
            want_raw = make_act_map_2d(&tm0, p.in0, p.fq.cin, p.S, p.T_in, p.fq.F_in, p.fq.T_raw0, p.fq.f_off0, nclips, pl.L.a_rows) &&
                       (!p.in1.x || make_act_map_2d(&tm1, p.in1, p.fq.cin, p.S, p.T_in, p.fq.F_in, p.fq.T_raw1, p.fq.f_off1, nclips, pl.L.a_rows));
        }
    }
    if (!want_raw) {
        pl = tc_plan(p, 4, false, g_deep_ring);
        if (!pl.ok) return cudaErrorInvalidConfiguration;
    }
    switch (p.n_tile) {
        case 16: return launch_tc_modes<16>(p, st, pl, n_tiles, freq, tm0, tm1);
        case 32: return launch_tc_modes<32>(p, st, pl, n_tiles, freq, tm0, tm1);
        case 64: return launch_tc_modes<64>(p, st, pl, n_tiles, freq, tm0, tm1);
        case 128:
            if (freq) return cudaErrorInvalidConfiguration;
            return (pair && want_raw) ? launch_tc_n<128, false, true>(p, st, pl, n_tiles, tm0, tm1)
                                      : launch_tc_n<128, false>(p, st, pl, n_tiles, tm0, tm1);
        default: return cudaErrorInvalidConfiguration;
    }
}

}  // namespace fcb
