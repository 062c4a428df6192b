// FreqCodec 2-D path (BASELINE config 4), first correct CUDA version: channels-last [B][F][T][C] SConv2d /
// SConvTranspose2d on the fp32 SIMT pipe, plus the STFT / iSTFT front and back ends with the mag_phase transforms.
//
// Reference: SConv2d / SConvTranspose2d / pad2d / unpad2d funcodec/modules/normed_modules/conv.py:102-141,317-447;
// FreqCodec._encode_frame / _decode_frame (mag_phase) funcodec/models/codec_freq.py:330-342,365-373,406-425,446-448;
// torchaudio Spectrogram / InverseSpectrogram defaults (n_fft 512, hop 160, periodic hann, center, reflect).
//
// The 2-D conv reuses the 1-D design (conv_simt.cu): every (clip, output frequency row) is a pseudo-clip of a 1-D conv
// along time whose input channels are the K_F frequency taps x C_in channels, gathered from K_F input rows while the
// tile is staged (reflect / zero indexing on both axes, deferred GroupNorm + resblock add + ELU on load).  A transposed
// conv (k = 2s per axis) is the 2x2-tap zero-padded conv with C_out' = s_f*s_t*C_out whose epilogue scatters phase
// (p_f, p_t) to row f*s_f + p_f, column t*s_t + p_t.  GroupNorm partials are emitted per pseudo-clip and summed per clip.
// These kernels are correctness-first (HBM- and FMA-bound rooflines as in conv_simt.cu); the tensor-core version is next.
#include "common.cuh"
#include "kernels.h"

namespace fcb {

template <int TX, int TM>
__global__ void __launch_bounds__(256, 2) conv2d_cl_kernel(const Conv2dParams p) {
    constexpr int TN = 8;
    constexpr int TY = 256 / TX;
    constexpr int CO_TILE = TX * TN;
    constexpr int T_TILE = TY * TM;
    extern __shared__ __align__(16) float smem[];
    const int tid = threadIdx.x;
    const int tx = tid % TX, ty = tid / TX;
    const int b = blockIdx.z / p.F_out, f_out = blockIdx.z - b * p.F_out;
    const int t0 = blockIdx.x * T_TILE;
    const int co0 = blockIdx.y * CO_TILE;
    const int C_in = p.C_in, cic = p.cic, KT = p.KT, ST = p.ST;
    const int R = (T_TILE - 1) * ST + (KT - 1) + 1;
    const int pitch = cic + 1;
    const bool has1 = p.in1.x != nullptr;

    float* Ws = smem;                                 // [KT][cic][CO_TILE]
    float* Xs = Ws + KT * cic * CO_TILE;              // [R][pitch]
    const float* cf0 = p.in0.coef ? p.in0.coef + (long long)b * 2 * C_in : nullptr;
    const float* cf1 = (has1 && p.in1.coef) ? p.in1.coef + (long long)b * 2 * C_in : nullptr;
    const int gt_max = (p.T_out - 1) * ST - p.pad_t + (KT - 1);

    float acc[TM][TN];
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

    const int c_st = tid % cic, r_st = tid / cic, r_step = 256 / cic;
    const int CK = p.KF * C_in;                      // gathered input channels

    for (int ci0 = 0; ci0 < CK; ci0 += cic) {
        __syncthreads();
        const int kfi = ci0 / C_in, cbase = ci0 - kfi * C_in;
        // frequency row of this tap
        int f_src = f_out * p.SF + kfi - p.pad_f;
        bool f_ok = true;
        if (p.pad_zero) f_ok = f_src >= 0 && f_src < p.F_in;
        else f_src = reflect_index(f_src, p.F_in);
        {
            const int c = cbase + c_st;
            float a0 = 1.f, b0 = 0.f, a1 = 1.f, b1 = 0.f;
            if (cf0) { a0 = __ldg(cf0 + c); b0 = __ldg(cf0 + C_in + c); }
            if (cf1) { a1 = __ldg(cf1 + c); b1 = __ldg(cf1 + C_in + c); }
            const float* x0 = p.in0.x + (((long long)b * p.in0.F_raw + p.in0.f_off + f_src) * p.in0.T_raw + p.in0.t_off) * C_in + c;
            const float* x1 = has1 ? p.in1.x + (((long long)b * p.in1.F_raw + p.in1.f_off + f_src) * p.in1.T_raw + p.in1.t_off) * C_in + c : nullptr;
            for (int row = r_st; row < R; row += r_step) {
                const int gt = t0 * ST - p.pad_t + row;
                float v = 0.f;
                bool ok = f_ok && gt <= gt_max;
                int src = gt;
                if (p.pad_zero) ok = ok && gt >= 0 && gt < p.T_in;
                else { src = reflect_index(gt, p.T_in); ok = ok && src >= 0 && src < p.T_in; }
                if (ok) {
                    v = fmaf(__ldg(x0 + (long long)src * C_in), a0, b0);
                    if (has1) v = v + fmaf(__ldg(x1 + (long long)src * C_in), a1, b1);
                    if (p.elu) v = elu1(v);
                }
                Xs[row * pitch + c_st] = v;
            }
        }
        for (int e = tid; e < KT * cic * CO_TILE; e += 256) {
            const int j = e % CO_TILE;
            const int kc = e / CO_TILE;
            const int k = kc / cic, c = kc - k * cic;
            const int co = co0 + j;
            Ws[e] = co < p.C_out_eff ? __ldg(p.w + ((long long)k * CK + ci0 + c) * p.C_out_eff + co) : 0.f;
        }
        __syncthreads();
        for (int c = 0; c < cic; ++c) {
            for (int k = 0; k < KT; ++k) {
                const float* xr = Xs + (ty * ST + k) * pitch + c;
                float a[TM];
#pragma unroll
                for (int i = 0; i < TM; ++i) a[i] = xr[i * TY * ST * pitch];
                const float* wrow = Ws + (k * cic + c) * CO_TILE + tx * 4;
                const float4 w0 = *reinterpret_cast<const float4*>(wrow);
                const float4 w1 = *reinterpret_cast<const float4*>(wrow + CO_TILE / 2);
#pragma unroll
                for (int i = 0; i < TM; ++i) {
                    acc[i][0] = fmaf(a[i], w0.x, acc[i][0]); acc[i][1] = fmaf(a[i], w0.y, acc[i][1]);
                    acc[i][2] = fmaf(a[i], w0.z, acc[i][2]); acc[i][3] = fmaf(a[i], w0.w, acc[i][3]);
                    acc[i][4] = fmaf(a[i], w1.x, acc[i][4]); acc[i][5] = fmaf(a[i], w1.y, acc[i][5]);
                    acc[i][6] = fmaf(a[i], w1.z, acc[i][6]); acc[i][7] = fmaf(a[i], w1.w, acc[i][7]);
                }
            }
        }
    }

    // ---- epilogue: bias, (phase-scattered) raw store, GroupNorm partial statistics
    float s = 0.f, ss = 0.f;
    const int coA = co0 + tx * 4, coB = co0 + CO_TILE / 2 + tx * 4;
    const int F2 = p.F_out * p.FR, T2 = p.T_out * p.TR;
#pragma unroll
    for (int i = 0; i < TM; ++i) {
        const int t = t0 + ty + i * TY;
        if (t >= p.T_out) continue;
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            const int co = half ? coB : coA;
            if (co >= p.C_out_eff) continue;
            // 4 consecutive output channels never straddle a phase boundary (Cc % 4 == 0)
            const int ph = co / p.Cc, cch = co - ph * p.Cc;
            const int pf = ph / p.TR, pt = ph - pf * p.TR;
            float* dst = p.out + (((long long)b * F2 + (long long)f_out * p.FR + pf) * T2 + (long long)t * p.TR + pt) * p.Cc + cch;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (co + j < p.C_out_eff) {
                    const float o = acc[i][4 * half + j] + __ldg(p.bias + co + j);
                    dst[j] = o;
                    s += o; ss = fmaf(o, o, ss);
                }
            }
        }
    }
    if (p.partials) {
        __shared__ double red[64];
        double ds = (double)s, dss = (double)ss;
        block_reduce_2d(ds, dss, red);
        if (tid == 0) {
            const int nparts = gridDim.x * gridDim.y;
            double* dst = p.partials + ((long long)blockIdx.z * nparts + blockIdx.y * gridDim.x + blockIdx.x) * 2;
            dst[0] = ds; dst[1] = dss;
        }
    }
}

static void conv2d_pick(const Conv2dParams& p, int* tx, int* tm) {
    *tx = p.C_out_eff >= 128 ? 16 : (p.C_out_eff >= 64 ? 8 : (p.C_out_eff >= 32 ? 4 : 2));
    *tm = 8;
    const int CO_TILE = *tx * 8, T_TILE = (256 / *tx) * 8;
    const long long ctas = (long long)((p.T_out + T_TILE - 1) / T_TILE) * ((p.C_out_eff + CO_TILE - 1) / CO_TILE) * p.B * p.F_out;
    if (ctas < 2 * 132) *tm = 4;
}

int conv2d_num_parts(const Conv2dParams& p) {
    int tx, tm;
    conv2d_pick(p, &tx, &tm);
    const int CO_TILE = tx * 8, T_TILE = (256 / tx) * tm;
    return ((p.T_out + T_TILE - 1) / T_TILE) * ((p.C_out_eff + CO_TILE - 1) / CO_TILE);
}

template <int TX, int TM>
static cudaError_t launch2d_cfg(Conv2dParams p, cudaStream_t st) {
    constexpr int CO_TILE = TX * 8, T_TILE = (256 / TX) * TM;
    int cic = 32;
    while (cic > 1 && (p.C_in % cic != 0)) cic >>= 1;
    auto bytes = [&](int c) {
        const int R = (T_TILE - 1) * p.ST + (p.KT - 1) + 1;
        return ((size_t)p.KT * c * CO_TILE + (size_t)R * (c + 1)) * sizeof(float);
    };
    while (cic > 1 && bytes(cic) > 100 * 1024) cic >>= 1;
    p.cic = cic;
    const size_t smem = bytes(cic);
    if (smem > 200 * 1024) return cudaErrorInvalidConfiguration;
    auto kern = conv2d_cl_kernel<TX, TM>;
    cudaError_t e = ensure_dynamic_smem((const void*)kern, 200 * 1024);
    if (e != cudaSuccess) return e;
    dim3 grid((p.T_out + T_TILE - 1) / T_TILE, (p.C_out_eff + CO_TILE - 1) / CO_TILE, p.B * p.F_out);
    kern<<<grid, 256, smem, st>>>(p);
    return cudaGetLastError();
}

cudaError_t launch_conv2d(const Conv2dParams& p, cudaStream_t st) {
    if (p.Cc % 4 != 0 && p.FR * p.TR > 1) return cudaErrorInvalidValue;
    int tx, tm;
    conv2d_pick(p, &tx, &tm);
#define FCB_CASE2(TX_, TM_) if (tx == TX_ && tm == TM_) return launch2d_cfg<TX_, TM_>(p, st);
    FCB_CASE2(2, 8) FCB_CASE2(2, 4) FCB_CASE2(4, 8) FCB_CASE2(4, 4) FCB_CASE2(8, 8) FCB_CASE2(8, 4) FCB_CASE2(16, 8) FCB_CASE2(16, 4)
#undef FCB_CASE2
    return cudaErrorInvalidConfiguration;
}

// =============================================================================================== small-C_out 2-D conv
// EXPERIMENTAL (option "conv2d_small_cout", off by default, not yet run on hardware): the 32 -> 3 (7 x 7) output conv of
// the FreqCodec decoder.  On the tensor-core path it wastes a 16-column n-tile on 3 outputs and re-transforms its input
// once per frequency tap (13.6 ms at config 4); here one CTA stages the normalised + ELU'd input ONCE as a
// (FT + K_F - 1) x (TT + K_T - 1) halo tile (8 channels at a time) and every thread keeps P = 5 adjacent time columns x
// C_out <= 4 outputs in registers, sliding along the K_T taps (10.8 FMA per shared-memory load: FMA-bound).
// Stride 1, reflect padding, no phase scatter.  Bound: fp32 FMA (38.8 GFMA per step at config 4).
constexpr int SC_FT = 8, SC_P = 5, SC_TT = 32 * SC_P, SC_CIC = 8, SC_CO = 4, SC_KMAX = 7;

__global__ void __launch_bounds__(256, 2) conv2d_small_cout_kernel(const Conv2dParams p) {
    extern __shared__ __align__(16) float smem[];
    const int tid = threadIdx.x;
    const int tg = tid & 31, fr = tid >> 5;                   // time group (P columns), frequency row of this thread
    const int b = blockIdx.z, f0 = blockIdx.y * SC_FT, t0 = blockIdx.x * SC_TT;
    const int KF = p.KF, KT = p.KT, C_in = p.C_in;
    const int HR = SC_FT + KF - 1, HC = SC_TT + KT - 1;       // halo rows / columns
    // Xs[c4 (2)][HR][HC] float4: a lane's window starts at column tg*P, so the lane-to-lane stride is P = 5 float4 (odd)
    // -> the 8 lanes of a quarter-warp hit 8 different 16-byte bank groups: conflict-free 128-bit reads without padding
    const int HCP = HC;
    float4* Xs = reinterpret_cast<float4*>(smem);
    float4* Ws = Xs + 2 * HR * HCP;                            // [KF][KT][c4 (2)][co (SC_CO)] float4 over the 4 channels of c4
    const bool has1 = p.in1.x != nullptr;
    const float* cf0 = p.in0.coef ? p.in0.coef + (long long)b * 2 * C_in : nullptr;
    const float* cf1 = (has1 && p.in1.coef) ? p.in1.coef + (long long)b * 2 * C_in : nullptr;
    const int CK = KF * C_in;

    float acc[SC_P][SC_CO];
#pragma unroll
    for (int i = 0; i < SC_P; ++i)
#pragma unroll
        for (int j = 0; j < SC_CO; ++j) acc[i][j] = 0.f;

    for (int ci0 = 0; ci0 < C_in; ci0 += SC_CIC) {
        __syncthreads();
        // ---- stage the halo tile of this channel chunk: deferred GroupNorm + resblock add + ELU applied once per element
        for (int e = tid; e < 2 * HR * HC; e += 256) {
            const int c4 = e & 1;
            const int rc = e >> 1;
            const int row = rc / HC, col = rc - row * HC;
            const int c = ci0 + c4 * 4;
            const int fs = reflect_index(f0 - p.pad_f + row, p.F_in);
            const int ts = reflect_index(t0 - p.pad_t + col, p.T_in);
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (fs >= 0 && fs < p.F_in && ts >= 0 && ts < p.T_in) {
                float4 a0 = make_float4(1.f, 1.f, 1.f, 1.f), b0 = make_float4(0.f, 0.f, 0.f, 0.f);
                if (cf0) { a0 = __ldg(reinterpret_cast<const float4*>(cf0 + c)); b0 = __ldg(reinterpret_cast<const float4*>(cf0 + C_in + c)); }
                const float4 x = __ldg(reinterpret_cast<const float4*>(
                    p.in0.x + (((long long)b * p.in0.F_raw + p.in0.f_off + fs) * p.in0.T_raw + p.in0.t_off + ts) * C_in + c));
                v.x = fmaf(x.x, a0.x, b0.x); v.y = fmaf(x.y, a0.y, b0.y); v.z = fmaf(x.z, a0.z, b0.z); v.w = fmaf(x.w, a0.w, b0.w);
                if (has1) {
                    float4 a1 = make_float4(1.f, 1.f, 1.f, 1.f), b1 = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (cf1) { a1 = __ldg(reinterpret_cast<const float4*>(cf1 + c)); b1 = __ldg(reinterpret_cast<const float4*>(cf1 + C_in + c)); }
                    const float4 y = __ldg(reinterpret_cast<const float4*>(
                        p.in1.x + (((long long)b * p.in1.F_raw + p.in1.f_off + fs) * p.in1.T_raw + p.in1.t_off + ts) * C_in + c));
                    v.x = v.x + fmaf(y.x, a1.x, b1.x); v.y = v.y + fmaf(y.y, a1.y, b1.y);
                    v.z = v.z + fmaf(y.z, a1.z, b1.z); v.w = v.w + fmaf(y.w, a1.w, b1.w);
                }
                if (p.elu) { v.x = elu1(v.x); v.y = elu1(v.y); v.z = elu1(v.z); v.w = elu1(v.w); }
            }
            Xs[(c4 * HR + row) * HCP + col] = v;
        }
        // ---- weights of this chunk: Ws[((kf*KT + kt)*2 + c4)*SC_CO + co] = W[kt][kf*C_in + ci0 + c4*4 .. +3][co]
        for (int e = tid; e < KF * KT * 2 * SC_CO; e += 256) {
            const int co = e % SC_CO;
            int r = e / SC_CO;
            const int c4 = r & 1; r >>= 1;
            const int kt = r % KT, kf = r / KT;
            float4 w = make_float4(0.f, 0.f, 0.f, 0.f);
            if (co < p.C_out_eff) {
                const float* wp = p.w + ((long long)kt * CK + kf * C_in + ci0 + c4 * 4) * p.C_out_eff + co;
                w.x = __ldg(wp); w.y = __ldg(wp + p.C_out_eff); w.z = __ldg(wp + 2 * p.C_out_eff); w.w = __ldg(wp + 3 * p.C_out_eff);
            }
            Ws[e] = w;
        }
        __syncthreads();
        // ---- compute: P sliding outputs x SC_CO channels per thread
        for (int kf = 0; kf < KF; ++kf) {
#pragma unroll
            for (int c4 = 0; c4 < 2; ++c4) {
                const float4* xr = Xs + (c4 * HR + fr + kf) * HCP;
                float4 x[SC_P + SC_KMAX - 1];
#pragma unroll
                for (int j = 0; j < SC_P + SC_KMAX - 1; ++j) {
                    x[j] = (j < SC_P + KT - 1) ? xr[tg * SC_P + j] : make_float4(0.f, 0.f, 0.f, 0.f);
                }
                const float4* wr = Ws + ((kf * KT) * 2 + c4) * SC_CO;
#pragma unroll
                for (int kt = 0; kt < SC_KMAX; ++kt) {
                    if (kt < KT) {
                        const float4 w0 = wr[kt * 2 * SC_CO + 0], w1 = wr[kt * 2 * SC_CO + 1], w2 = wr[kt * 2 * SC_CO + 2],
                                     w3 = wr[kt * 2 * SC_CO + 3];
#pragma unroll
                        for (int i = 0; i < SC_P; ++i) {
                            const float4 xv = x[i + kt];
                            acc[i][0] = fmaf(xv.x, w0.x, acc[i][0]); acc[i][0] = fmaf(xv.y, w0.y, acc[i][0]);
                            acc[i][0] = fmaf(xv.z, w0.z, acc[i][0]); acc[i][0] = fmaf(xv.w, w0.w, acc[i][0]);
                            acc[i][1] = fmaf(xv.x, w1.x, acc[i][1]); acc[i][1] = fmaf(xv.y, w1.y, acc[i][1]);
                            acc[i][1] = fmaf(xv.z, w1.z, acc[i][1]); acc[i][1] = fmaf(xv.w, w1.w, acc[i][1]);
                            acc[i][2] = fmaf(xv.x, w2.x, acc[i][2]); acc[i][2] = fmaf(xv.y, w2.y, acc[i][2]);
                            acc[i][2] = fmaf(xv.z, w2.z, acc[i][2]); acc[i][2] = fmaf(xv.w, w2.w, acc[i][2]);
                            acc[i][3] = fmaf(xv.x, w3.x, acc[i][3]); acc[i][3] = fmaf(xv.y, w3.y, acc[i][3]);
                            acc[i][3] = fmaf(xv.z, w3.z, acc[i][3]); acc[i][3] = fmaf(xv.w, w3.w, acc[i][3]);
                        }
                    }
                }
            }
        }
    }

    // ---- epilogue: bias, raw store of the real channels, GroupNorm partial statistics
    float s = 0.f, ss = 0.f;
    const int f = f0 + fr;
    if (f < p.F_out) {
#pragma unroll
        for (int i = 0; i < SC_P; ++i) {
            const int t = t0 + tg * SC_P + i;
            if (t >= p.T_out) continue;
            float* dst = p.out + (((long long)b * p.F_out + f) * p.T_out + t) * p.C_out_eff;
#pragma unroll
            for (int co = 0; co < SC_CO; ++co) {
                if (co < p.C_out_eff) {
                    const float o = acc[i][co] + __ldg(p.bias + co);
                    dst[co] = o;
                    s += o; ss = fmaf(o, o, ss);
                }
            }
        }
    }
    if (p.partials) {
        __shared__ double red[64];
        double ds = (double)s, dss = (double)ss;
        block_reduce_2d(ds, dss, red);
        if (tid == 0) {
            const int nparts = gridDim.x * gridDim.y;
            double* dst = p.partials + ((long long)b * nparts + blockIdx.y * gridDim.x + blockIdx.x) * 2;
            dst[0] = ds; dst[1] = dss;
        }
    }
}

bool conv2d_small_cout_supported(const Conv2dParams& p) {
    return p.SF == 1 && p.ST == 1 && p.FR == 1 && p.TR == 1 && !p.pad_zero && p.C_out_eff <= SC_CO && p.C_in % SC_CIC == 0 &&
           p.KF <= SC_KMAX && p.KT <= SC_KMAX && p.F_out == p.F_in && p.T_out == p.T_in;
}

// partial statistics per clip (the caller passes B * this many (sum, sum^2) pairs)
int conv2d_small_cout_num_parts(const Conv2dParams& p) {
    return ((p.T_out + SC_TT - 1) / SC_TT) * ((p.F_out + SC_FT - 1) / SC_FT);
}

cudaError_t launch_conv2d_small_cout(const Conv2dParams& p, cudaStream_t st) {
    if (!conv2d_small_cout_supported(p)) return cudaErrorInvalidValue;
    const int HR = SC_FT + p.KF - 1, HC = SC_TT + p.KT - 1, HCP = HC;
    const size_t smem = ((size_t)2 * HR * HCP + (size_t)p.KF * p.KT * 2 * SC_CO) * sizeof(float4);
    cudaError_t e = ensure_dynamic_smem((const void*)conv2d_small_cout_kernel, 110 * 1024);
    if (e != cudaSuccess) return e;
    if (smem > 110 * 1024) return cudaErrorInvalidConfiguration;
    dim3 grid((p.T_out + SC_TT - 1) / SC_TT, (p.F_out + SC_FT - 1) / SC_FT, p.B);
    conv2d_small_cout_kernel<<<grid, 256, smem, st>>>(p);
    return cudaGetLastError();
}

// =============================================================================================== STFT front end
// One CTA = 8 frames of one clip.  X[k] = sum_n (x[n]/scale) w[n] e^{-2 pi i k n / N}, then the mag_phase features
// (codec_freq.py:365-373) written channels-last as [B][N/2+1][T_s][cpad] = (log max(|X|,1e-6), Re X/max(|X|,1e-6), Im ...)
// followed by cpad - 3 zero channels (cpad = 4: one element is one aligned 16-byte load for the first conv).
constexpr int STFT_FR = 8;

__global__ void __launch_bounds__(256) stft_magphase_kernel(const float* __restrict__ wav, const float* __restrict__ scale, int L,
                                                            int n_fft, int hop, int n_frames, int cpad, float* __restrict__ feats) {
    extern __shared__ __align__(16) float smem[];
    float* cs = smem;                 // [n_fft] cos(2 pi j / N)
    float* sn = cs + n_fft;           // [n_fft] sin(2 pi j / N)
    float* win = sn + n_fft;          // [n_fft] periodic hann
    float* xs = win + n_fft;          // [n_fft + (STFT_FR-1)*hop] samples of this frame group
    const int b = blockIdx.y, fr0 = blockIdx.x * STFT_FR;
    const int tid = threadIdx.x;
    for (int j = tid; j < n_fft; j += 256) {
        float s, c;
        sincospif(2.0f * (float)j / (float)n_fft, &s, &c);
        cs[j] = c; sn[j] = s;
        win[j] = 0.5f - 0.5f * c;
    }
    const int span = n_fft + (STFT_FR - 1) * hop;
    const float sc = scale ? scale[b] : 1.0f;
    for (int i = tid; i < span; i += 256) {
        const int g = fr0 * hop - n_fft / 2 + i;          // center=True: frame m covers [m*hop - N/2, m*hop + N/2)
        const int src = reflect_index(g, L);
        float v = 0.f;
        if (src >= 0 && src < L) v = wav[(long long)b * L + src] / sc;
        xs[i] = v;
    }
    __syncthreads();
    const int n_bins = n_fft / 2 + 1;
    for (int o = tid; o < n_bins * STFT_FR; o += 256) {
        const int fi = o / n_bins, k = o - fi * n_bins;
        const int m = fr0 + fi;
        if (m >= n_frames) continue;
        const float* xf = xs + fi * hop;
        float re = 0.f, im = 0.f;
        int idx = 0;                                       // (k * n) mod n_fft, incrementally
        for (int n = 0; n < n_fft; ++n) {
            const float xw = xf[n] * win[n];
            re = fmaf(xw, cs[idx], re);
            im = fmaf(-xw, sn[idx], im);
            idx += k;
            if (idx >= n_fft) idx -= n_fft;
        }
        const float mag = hypotf(re, im);
        const float cl = fmaxf(mag, 1e-6f);
        float* dst = feats + (((long long)b * n_bins + k) * n_frames + m) * cpad;
        dst[0] = logf(cl);
        dst[1] = re / cl;
        dst[2] = im / cl;
        for (int c = 3; c < cpad; ++c) dst[c] = 0.f;
    }
}

cudaError_t launch_stft_magphase(const float* wav, const float* scale, int B, int L, int n_fft, int hop, int n_frames,
                                 int cpad, float* feats, cudaStream_t st) {
    if (cpad < 3) return cudaErrorInvalidValue;
    const size_t smem = ((size_t)4 * n_fft + (STFT_FR - 1) * hop) * sizeof(float);
    cudaError_t e = ensure_dynamic_smem((const void*)stft_magphase_kernel, 100 * 1024);
    if (e != cudaSuccess) return e;
    stft_magphase_kernel<<<dim3((n_frames + STFT_FR - 1) / STFT_FR, B), 256, smem, st>>>(wav, scale, L, n_fft, hop, n_frames, cpad, feats);
    return cudaGetLastError();
}

// ----------------------------------------------------------------------------------------------- STFT as a GEMM
// EXPERIMENTAL (option "stft_tc", off by default, not yet run on hardware): X = frames x DFT basis on the tensor-core conv
// kernel.  With hop and n_fft multiples of 32 the padded waveform viewed as rows of 32 samples [Lp/32][32] is a
// channels-last tensor, and frame m = rows 5m .. 5m+15 (hop 160, n_fft 512): a k = n_fft/32, s = hop/32 conv with
// C_out = 2*(n_fft/2+1) basis columns (window folded in).  The kernels below are the glue: padded/scaled rows in,
// (re, im) columns -> mag_phase features out.
__global__ void wave_rows_kernel(const float* __restrict__ wav, const float* __restrict__ scale, int L, int n_fft, long long n_out,
                                 float* __restrict__ rows) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;          // sample of the padded signal
    const int b = blockIdx.y;
    if (i >= n_out) return;
    const int src = reflect_index((int)i - n_fft / 2, L);                            // center=True, pad_mode="reflect"
    float v = 0.f;
    if (src >= 0 && src < L && i < (long long)L + n_fft) v = wav[(long long)b * L + src] / (scale ? scale[b] : 1.0f);
    rows[(long long)b * n_out + i] = v;
}

cudaError_t launch_wave_rows(const float* wav, const float* scale, int B, int L, int n_fft, int n_rows, float* rows, cudaStream_t st) {
    const long long n_out = (long long)n_rows * 32;
    wave_rows_kernel<<<dim3((unsigned)((n_out + 255) / 256), B), 256, 0, st>>>(wav, scale, L, n_fft, n_out, rows);
    return cudaGetLastError();
}

// spec [B][T_s][ld] with Re X[k] in column k and Im X[k] in column n_bins + k  ->  feats [B][n_bins][T_s][cpad]
// (32 x 32 shared-memory transpose: coalesced on both sides)
__global__ void magphase_from_spec_kernel(const float* __restrict__ spec, int ld, int n_bins, int n_frames, int cpad,
                                          float* __restrict__ feats) {
    __shared__ float re[32][33], im[32][33];
    const int b = blockIdx.z, k0 = blockIdx.x * 32, m0 = blockIdx.y * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;                          // 256 threads: 8 rows per pass
    for (int r = ty; r < 32; r += 8) {
        const int m = m0 + r, k = k0 + tx;
        float a = 0.f, c = 0.f;
        if (m < n_frames && k < n_bins) {
            const float* sp = spec + ((long long)b * n_frames + m) * ld;
            a = sp[k]; c = sp[n_bins + k];
        }
        re[r][tx] = a; im[r][tx] = c;
    }
    __syncthreads();
    for (int r = ty; r < 32; r += 8) {
        const int k = k0 + r, m = m0 + tx;
        if (k < n_bins && m < n_frames) {
            const float xr = re[tx][r], xi = im[tx][r];
            const float mag = hypotf(xr, xi);
            const float cl = fmaxf(mag, 1e-6f);
            float* dst = feats + (((long long)b * n_bins + k) * n_frames + m) * cpad;
            dst[0] = logf(cl); dst[1] = xr / cl; dst[2] = xi / cl;
            for (int c = 3; c < cpad; ++c) dst[c] = 0.f;
        }
    }
}

cudaError_t launch_magphase_from_spec(const float* spec, int ld, int B, int n_bins, int n_frames, int cpad, float* feats,
                                      cudaStream_t st) {
    magphase_from_spec_kernel<<<dim3((n_bins + 31) / 32, (n_frames + 31) / 32, B), 256, 0, st>>>(spec, ld, n_bins, n_frames, cpad, feats);
    return cudaGetLastError();
}

// decoder output raw [B][F_raw][T_raw][3] (+ deferred GroupNorm coef) -> Y [B][n_frames][ld]: column k = softplus(mag) * re,
// column n_bins + k = softplus(mag) * im (codec_freq.py:417-425), zero beyond 2*n_bins: the A operand of the iSTFT GEMM
__global__ void spec_rows_kernel(const float* __restrict__ raw, const float* __restrict__ coef, int F_raw, int T_raw, int n_bins,
                                 int n_frames, int ld, float* __restrict__ Y) {
    __shared__ float yr[32][33], yi[32][33];
    const int b = blockIdx.z, k0 = blockIdx.x * 32, m0 = blockIdx.y * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const float* cf = coef + (long long)b * 6;
    for (int r = ty; r < 32; r += 8) {
        const int k = k0 + r, m = m0 + tx;
        float a = 0.f, c = 0.f;
        if (k < n_bins && m < n_frames) {
            const float* src = raw + (((long long)b * F_raw + k) * T_raw + m) * 3;
            const float y0 = fmaf(src[0], cf[0], cf[3]);
            const float y1 = fmaf(src[1], cf[1], cf[4]);
            const float y2 = fmaf(src[2], cf[2], cf[5]);
            const float mag = y0 > 20.f ? y0 : log1pf(expf(y0));
            a = mag * y1; c = mag * y2;
        }
        yr[r][tx] = a; yi[r][tx] = c;
    }
    __syncthreads();
    for (int r = ty; r < 32; r += 8) {
        const int m = m0 + r, k = k0 + tx;
        if (m < n_frames && k < n_bins) {
            float* dst = Y + ((long long)b * n_frames + m) * ld;
            dst[k] = yr[tx][r];
            dst[n_bins + k] = yi[tx][r];
        }
    }
}

cudaError_t launch_spec_rows(const float* raw, const float* coef, int B, int F_raw, int T_raw, int n_bins, int n_frames, int ld,
                             float* Y, cudaStream_t st) {
    cudaError_t e = cudaMemsetAsync(Y, 0, (size_t)B * n_frames * ld * sizeof(float), st);     // the padding columns
    if (e != cudaSuccess) return e;
    spec_rows_kernel<<<dim3((n_bins + 31) / 32, (n_frames + 31) / 32, B), 256, 0, st>>>(raw, coef, F_raw, T_raw, n_bins, n_frames, ld, Y);
    return cudaGetLastError();
}

// =============================================================================================== iSTFT back end
// Frame synthesis: (deferred GroupNorm of the decoder's last conv) -> softplus(mag) * (re + i im) (codec_freq.py:417-425)
// -> irfft (DC / Nyquist imaginary parts ignored) -> x hann window, one CTA per (frame, clip) -> frames [B][T_s][N].
__global__ void __launch_bounds__(256) istft_frames_kernel(const float* __restrict__ raw, const float* __restrict__ coef, int F_raw,
                                                           int T_raw, int n_fft, int n_frames, float* __restrict__ frames) {
    extern __shared__ __align__(16) float smem[];
    float* cs = smem;
    float* sn = cs + n_fft;
    float* xr = sn + n_fft;           // [n_bins] Re X
    float* xi = xr + n_fft / 2 + 1;   // [n_bins] Im X
    const int m = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
    const int n_bins = n_fft / 2 + 1;
    for (int j = tid; j < n_fft; j += 256) {
        float s, c;
        sincospif(2.0f * (float)j / (float)n_fft, &s, &c);
        cs[j] = c; sn[j] = s;
    }
    const float* cf = coef + (long long)b * 6;           // [2][3]: a0 a1 a2 b0 b1 b2
    for (int k = tid; k < n_bins; k += 256) {
        const float* src = raw + (((long long)b * F_raw + k) * T_raw + m) * 3;
        const float y0 = fmaf(src[0], cf[0], cf[3]);
        const float y1 = fmaf(src[1], cf[1], cf[4]);
        const float y2 = fmaf(src[2], cf[2], cf[5]);
        const float mag = y0 > 20.f ? y0 : log1pf(expf(y0));      // F.softplus(beta=1, threshold=20)
        xr[k] = mag * y1;
        xi[k] = mag * y2;
    }
    __syncthreads();
    const float inv_n = 1.0f / (float)n_fft;
    for (int j = tid; j < n_fft; j += 256) {
        float acc = 0.f;
        int idx = j;                                               // (k * j) mod n_fft for k = 1
        for (int k = 1; k < n_bins - 1; ++k) {
            acc = fmaf(xr[k], cs[idx], acc);
            acc = fmaf(-xi[k], sn[idx], acc);
            idx += j;
            if (idx >= n_fft) idx -= n_fft;
        }
        const float nyq = (j & 1) ? -xr[n_bins - 1] : xr[n_bins - 1];
        const float v = (xr[0] + nyq + 2.0f * acc) * inv_n;
        const float w = 0.5f - 0.5f * cs[j];
        frames[((long long)b * n_frames + m) * n_fft + j] = v * w;
    }
}

// Overlap-add, window-envelope normalisation, center trim, optional * scale, keep out_len samples (torch.istft + the
// reference's `[:, :, :L]`).
__global__ void istft_ola_kernel(const float* __restrict__ frames, const float* __restrict__ scale, int n_fft, int hop, int n_frames,
                                 int out_len, float* __restrict__ out) {
    const int b = blockIdx.y;
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= out_len) return;
    const int np = n + n_fft / 2;
    int m_hi = np / hop;
    if (m_hi > n_frames - 1) m_hi = n_frames - 1;
    float acc = 0.f, env = 0.f;
    for (int m = m_hi; m >= 0; --m) {
        const int j = np - m * hop;
        if (j >= n_fft) break;
        float s, c;
        sincospif(2.0f * (float)j / (float)n_fft, &s, &c);
        const float w = 0.5f - 0.5f * c;
        acc += frames[((long long)b * n_frames + m) * n_fft + j];
        env = fmaf(w, w, env);
    }
    float v = acc / env;
    if (scale) v *= scale[b];
    out[(long long)b * out_len + n] = v;
}

cudaError_t launch_istft_ola(const float* frames, const float* scale, int B, int n_fft, int hop, int n_frames, int out_len,
                             float* out, cudaStream_t st) {
    istft_ola_kernel<<<dim3((out_len + 255) / 256, B), 256, 0, st>>>(frames, scale, n_fft, hop, n_frames, out_len, out);
    return cudaGetLastError();
}

cudaError_t launch_istft(const float* raw, const float* coef, int B, int F_raw, int T_raw, int n_fft, int hop, int n_frames,
                         const float* scale, float* frames, float* out, int out_len, cudaStream_t st) {
    const size_t smem = ((size_t)2 * n_fft + 2 * (n_fft / 2 + 1)) * sizeof(float);
    istft_frames_kernel<<<dim3(n_frames, B), 256, smem, st>>>(raw, coef, F_raw, T_raw, n_fft, n_frames, frames);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    istft_ola_kernel<<<dim3((out_len + 255) / 256, B), 256, 0, st>>>(frames, scale, n_fft, hop, n_frames, out_len, out);
    return cudaGetLastError();
}

}  // namespace fcb
