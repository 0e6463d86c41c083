// Streaming decimating FIR — the H100 replacement for the `filter` block's per-cycle module chain
// (src/domains/dsp/filter/block_impl.cc:350-582): pad -> fft -> multiply(filter spectrum) -> fold ->
// ifft -> multiply_constant(1/M) -> unpad -> overlap_add.
//
// That chain computes, frame by frame with a carried tail, exactly the causal linear convolution of the
// time-continuous stream (the batch axis holds consecutive frames, overlap_add/module_impl_native_cpu.cc:155-198)
// with the taps, kept at every R-th sample when the block resamples (fold + ifft + 1/M == time-domain
// decimation, SURVEY.md Appendix B):
//        y[q] = sum_{k=0}^{L-1} h[k] * xs[q R - k],      xs = ... previous cycles ..., frame 0, frame 1, ...
// so it is evaluated directly in the time domain: one pass over the input (8 B/sample), 8/R B/sample out,
// state = the last L-1 input samples (instead of the reference's (L-1)/R output-tail samples).
//
// Kernel: a CTA stages the input span of a tile of QT = threads*OB outputs into shared memory, split into
// R polyphase planes (plane p holds xs[.. + p], unit stride in q, odd plane pitch: conflict-free); each
// thread owns OB consecutive outputs and walks the taps of one plane at a time with a register sliding
// window (1 shared load + 2 OB FMAs per tap), so the FP32 pipe, not shared memory, is the inner
// bound. Taps are re-ordered per plane on the host and live in shared memory (broadcast loads).
#include <algorithm>
#include <cmath>
#include <complex>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <type_traits>
#include <vector>

#include "common.cuh"

namespace b200 {

constexpr uint32_t kFirConstTapWords = 1024;     // tap tables up to 4 KB travel in the kernel parameters (constant bank)

struct FirParams {
    const float2* x;        // [n_in] stream (frames concatenated)
    const float2* hist;     // [L-1] last inputs of the previous call (zeros initially)
    float2* y;              // [frames, heads, frame_out]
    const float* taps;      // device: [heads][R][lp_pad] real, or complex as float2
    uint64_t n_in, n_out;   // n_out = n_in / R
    uint32_t L, R, heads;
    uint32_t lp_pad;        // taps per plane, padded to a multiple of OB
    uint32_t hpad;          // history rows (in units of R samples) staged below the tile, incl. OB slack
    uint32_t qt;            // outputs per tile = blockDim.x * OB
    uint32_t plane_pitch;   // chosen so one warp's cp.async scatter over the planes is bank-conflict-free
    uint32_t lp;            // taps of plane 0 = ceil(L / R); planes with kp0 >= lp_thr hold lp - 1
    uint32_t lp_thr;
    uint64_t frame_out;     // outputs per frame (T / R)
    // Frequency-translating heads (resampling with a non-zero centre): y is multiplied by
    // rot[head][m] * corr[head][frame]  (fold offsets + phase_correction of the reference), else nullptr.
    const float2* rot;      // [heads, frame_out]   exp(-j 2 pi c_h (m R) / M), F64-evaluated
    const float2* corr;     // [heads, frames]      exp(j (phase_h + inc_h frame)), F64-evaluated per call
    uint64_t frames;
    // CONST_TAPS: the re-ordered tap table itself. Tap reads then go through the constant cache (LDC) instead of the
    // shared-memory pipe, which the sliding-window loads already keep two thirds busy.
    float taps_c[kFirConstTapWords];
};

// PAIR (even R, odd L, even stream length, 16-byte aligned stream; real or complex taps): the same algorithm on 16-byte CHUNKS
// c[n] = (x[2n], x[2n+1]) with decimation R / 2 and chunk-taps g[c] = (h[2c], h[2c-1]):
//        y[q] = sum_c  h[2c] * x[qR - 2c]  +  h[2c-1] * x[qR - 2c + 1]  =  sum_c g[c] . chunk[q R/2 - c],
// i.e. every p.* field below is in chunk units (p.R = R/2, p.L = (L+1)/2, p.n_in = n_in/2). One LDGSTS.128 stages two
// samples and one LDS.128 feeds 4 OB FMAs: half the staging and window-load instructions of the 8-byte form.
template <uint32_t BYTES>
__device__ __forceinline__ void cp_async_elem(const uint32_t dst, const void* src) {
    if constexpr (BYTES == 16) {
        asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
    } else {
        asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(dst), "l"(src) : "memory");
    }
}
template <uint32_t BYTES>
__device__ __forceinline__ void cp_async_elem_fill(const uint32_t dst, const void* src, const uint32_t bytes) {
    if constexpr (BYTES == 16) {
        asm volatile("cp.async.ca.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(bytes) : "memory");
    } else {
        asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;" ::"r"(dst), "l"(src), "r"(bytes) : "memory");
    }
}

template <int OB, bool REAL_TAPS, bool CONST_TAPS, bool PAIR = false>
__global__ void __launch_bounds__(128) fir_decim_kernel(const __grid_constant__ FirParams p) {
    using E = typename std::conditional<PAIR, float4, float2>::type;     // staged element
    constexpr uint32_t EB = sizeof(E);
    constexpr int TW = (PAIR ? 2 : 1) * (REAL_TAPS ? 1 : 2);             // floats per tap slot
    extern __shared__ __align__(16) unsigned char smem_raw[];
    E* const planes = reinterpret_cast<E*>(smem_raw);
    const E* const xsrc = reinterpret_cast<const E*>(p.x);
    const E* const hsrc = reinterpret_cast<const E*>(p.hist);
    const uint32_t tap_words = p.heads * p.R * p.lp_pad * TW;
    float* const taps_s = reinterpret_cast<float*>(planes + static_cast<size_t>(p.R) * p.plane_pitch);
    float2* const out_s = reinterpret_cast<float2*>(taps_s + ((tap_words + 1) & ~1u));

    const uint32_t tid = threadIdx.x, nthreads = blockDim.x;
    if constexpr (!CONST_TAPS) {
        for (uint32_t i = tid; i < tap_words; i += nthreads) {
            taps_s[i] = p.taps[i];
        }
    }

    const uint64_t tiles = (p.n_out + p.qt - 1) / p.qt;
    const uint32_t span = (p.qt - 1) * p.R + p.hpad * p.R + 1;     // staged samples per tile
    const int64_t hist_len = static_cast<int64_t>(p.L) - 1;

    for (uint64_t tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const uint64_t q0 = tile * p.qt;
        const int64_t j0 = static_cast<int64_t>(q0 * p.R) - static_cast<int64_t>(p.hpad) * p.R;
        __syncthreads();   // previous tile's out_s/planes consumers are done
        // ---- stage: sample i (stream index j0 + i) -> plane[i mod R][i div R] with cp.async (LDGSTS, 8 bytes):
        // every request of the tile is in flight at once and no register is held for it. Out-of-range samples
        // are zero-filled by the src-size operand. (Versions that waited per load / per batch of 8 were
        // long-scoreboard bound.)
        {
            uint32_t plane = tid % p.R, pos = tid / p.R;
            const uint32_t step_plane = nthreads % p.R, step_pos = nthreads / p.R;
            const uint32_t plane_base = static_cast<uint32_t>(__cvta_generic_to_shared(planes));
            const bool interior = j0 >= 0 && static_cast<uint64_t>(j0) + span <= p.n_in;   // CTA-uniform
            if (interior && step_plane == 0) {
                // nthreads % R == 0: a thread stays on one plane, source and destination advance by constants
                // (3 instructions per request instead of 22 in the generic loop, which was 38 % of all
                // instructions issued by the first version).
                const E* src = xsrc + j0 + tid;
                uint32_t dst = plane_base + (plane * p.plane_pitch + pos) * EB;
                const uint32_t dst_step = step_pos * EB;
                uint32_t i = tid;
                for (; i + 3 * nthreads < span; i += 4 * nthreads) {
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        cp_async_elem<EB>(dst + u * dst_step, src + u * nthreads);
                    }
                    src += 4 * nthreads;
                    dst += 4 * dst_step;
                }
                for (; i < span; i += nthreads) {
                    cp_async_elem<EB>(dst, src);
                    src += nthreads;
                    dst += dst_step;
                }
            } else if (interior) {
                const E* src = xsrc + j0 + tid;
                for (uint32_t i = tid; i < span; i += nthreads) {
                    const uint32_t dst = plane_base + (plane * p.plane_pitch + pos) * EB;
                    cp_async_elem<EB>(dst, src);
                    src += nthreads;
                    plane += step_plane;
                    pos += step_pos;
                    if (plane >= p.R) {
                        plane -= p.R;
                        ++pos;
                    }
                }
            } else {
                for (uint32_t i = tid; i < span; i += nthreads) {
                    const int64_t j = j0 + i;
                    const E* src = xsrc;
                    uint32_t bytes = 0;
                    if (j >= 0) {
                        if (static_cast<uint64_t>(j) < p.n_in) {
                            src = xsrc + j;
                            bytes = EB;
                        }
                    } else if (j >= -hist_len) {
                        src = hsrc + (hist_len + j);
                        bytes = EB;
                    }
                    const uint32_t dst = plane_base + (plane * p.plane_pitch + pos) * EB;
                    cp_async_elem_fill<EB>(dst, src, bytes);
                    plane += step_plane;
                    pos += step_pos;
                    if (plane >= p.R) {
                        plane -= p.R;
                        ++pos;
                    }
                }
            }
            asm volatile("cp.async.commit_group;" ::: "memory");
            asm volatile("cp.async.wait_group 0;" ::: "memory");
        }
        __syncthreads();

        const uint32_t o0 = tid * OB;
        for (uint32_t head = 0; head < p.heads; ++head) {
            float2 acc[OB];
#pragma unroll
            for (int i = 0; i < OB; ++i) {
                acc[i] = make_float2(0.f, 0.f);
            }
            for (uint32_t plane = 0; plane < p.R; ++plane) {
                // taps of this plane: k = kp0 + m R with kp0 = (R - plane) % R; input row offset D - m
                const uint32_t d = plane == 0 ? p.hpad : p.hpad - 1;
                const E* const xp = planes + static_cast<size_t>(plane) * p.plane_pitch + o0 + d;
                const float* const hp = taps_s + (static_cast<size_t>(head) * p.R + plane) * p.lp_pad * TW;
                E w[OB];
#pragma unroll
                for (int i = 0; i < OB; ++i) {
                    w[i] = xp[i];
                }
                const E* xq = xp;           // xq[-(s+1)] is the element tap (m0 + s + 1) slides in
                const float* hq = hp;
                uint32_t hc = (head * p.R + plane) * p.lp_pad * TW;     // index into p.taps_c
                // taps actually present in this plane: k = kp0 + m R < L  (the padded tail is skipped, not multiplied)
                const uint32_t kp0 = plane == 0 ? 0 : p.R - plane;
                const uint32_t lp_plane = p.lp - (kp0 >= p.lp_thr ? 1u : 0u);      // == ceil((L - kp0) / R), no division
                const uint32_t full = lp_plane / OB * OB;
                auto tap_step = [&](const int s) {
                    // logical window element i lives in w[(i - s) mod OB]
                    if constexpr (PAIR && REAL_TAPS) {
                        const float ha = CONST_TAPS ? p.taps_c[hc + 2 * s] : hq[2 * s];
                        const float hb = CONST_TAPS ? p.taps_c[hc + 2 * s + 1] : hq[2 * s + 1];
                        const float2 ga = make_float2(ha, ha), gb = make_float2(hb, hb);
#pragma unroll
                        for (int i = 0; i < OB; ++i) {
                            const float4 v = w[(i - s + OB) % OB];
                            acc[i] = ffma2(make_float2(v.x, v.y), ga, acc[i]);
                            acc[i] = ffma2(make_float2(v.z, v.w), gb, acc[i]);
                        }
                    } else if constexpr (PAIR) {
                        // complex chunk-taps (frequency-translating heads): (h[2c], h[2c-1]) as four floats
                        const float ar = CONST_TAPS ? p.taps_c[hc + 4 * s] : hq[4 * s];
                        const float ai = CONST_TAPS ? p.taps_c[hc + 4 * s + 1] : hq[4 * s + 1];
                        const float br = CONST_TAPS ? p.taps_c[hc + 4 * s + 2] : hq[4 * s + 2];
                        const float bi = CONST_TAPS ? p.taps_c[hc + 4 * s + 3] : hq[4 * s + 3];
                        const float2 gar = make_float2(ar, ar), gai = make_float2(-ai, ai);
                        const float2 gbr = make_float2(br, br), gbi = make_float2(-bi, bi);
#pragma unroll
                        for (int i = 0; i < OB; ++i) {
                            const float4 v = w[(i - s + OB) % OB];
                            acc[i] = ffma2(make_float2(v.x, v.y), gar, acc[i]);
                            acc[i] = ffma2(make_float2(v.y, v.x), gai, acc[i]);
                            acc[i] = ffma2(make_float2(v.z, v.w), gbr, acc[i]);
                            acc[i] = ffma2(make_float2(v.w, v.z), gbi, acc[i]);
                        }
                    } else if constexpr (REAL_TAPS) {
                        const float h = CONST_TAPS ? p.taps_c[hc + s] : hq[s];
                        const float2 hh = make_float2(h, h);
#pragma unroll
                        for (int i = 0; i < OB; ++i) {
                            acc[i] = ffma2(w[(i - s + OB) % OB], hh, acc[i]);
                        }
                    } else {
                        const float2 h = CONST_TAPS ? make_float2(p.taps_c[hc + 2 * s], p.taps_c[hc + 2 * s + 1])
                                                    : reinterpret_cast<const float2*>(hq)[s];
                        const float2 hr = make_float2(h.x, h.x), hi = make_float2(-h.y, h.y);
#pragma unroll
                        for (int i = 0; i < OB; ++i) {
                            const float2 v = w[(i - s + OB) % OB];
                            acc[i] = ffma2(v, hr, acc[i]);
                            acc[i] = ffma2(make_float2(v.y, v.x), hi, acc[i]);
                        }
                    }
                    // slide: next tap (m+1) needs row offset one lower
                    w[(OB - 1 - s) % OB] = xq[-s - 1];
                };
                for (uint32_t m0 = 0; m0 < full; m0 += OB) {
#pragma unroll
                    for (int s = 0; s < OB; ++s) {
                        tap_step(s);
                    }
                    xq -= OB;
                    hq += OB * TW;
                    hc += OB * TW;
                }
                const uint32_t rem = lp_plane - full;       // CTA-uniform
#pragma unroll
                for (int s = 0; s < OB - 1; ++s) {
                    if (static_cast<uint32_t>(s) < rem) {
                        tap_step(s);
                    }
                }
            }
            // ---- stage the tile's outputs, then store coalesced
            __syncthreads();
#pragma unroll
            for (int i = 0; i < OB; ++i) {
                out_s[o0 + i] = acc[i];
            }
            __syncthreads();
            if (p.heads == 1 && p.rot == nullptr) {
                for (uint32_t o = tid; o < p.qt; o += nthreads) {
                    if (q0 + o < p.n_out) {
                        stg_stream_f2(p.y + q0 + o, out_s[o]);      // [frames, 1, frame_out] is the stream itself
                    }
                }
            } else {
                uint64_t frame = (q0 + tid) / p.frame_out;
                uint64_t m = (q0 + tid) - frame * p.frame_out;
                for (uint32_t o = tid; o < p.qt; o += nthreads) {
                    if (q0 + o < p.n_out) {
                        float2 v = out_s[o];
                        if (p.rot != nullptr) {
                            v = cmul_exact(cmul_exact(v, p.rot[head * p.frame_out + m]), p.corr[head * p.frames + frame]);
                        }
                        stg_stream_f2(p.y + (frame * p.heads + head) * p.frame_out + m, v);
                    }
                    m += nthreads;
                    while (m >= p.frame_out) {
                        m -= p.frame_out;
                        ++frame;
                    }
                }
            }
        }
    }
}

// phase_correction (src/domains/dsp/phase_correction/module_impl_native_cpu.cc:81-115): per head and frame the
// phasor exp(j (phase_h + inc_h * frame)) in F64 -> F32; afterwards phase_h <- remainder(phase_h + inc_h * frames, 2 pi).
__global__ void fir_frame_corr_kernel(float2* __restrict__ corr, double* __restrict__ phases,
                                      const double* __restrict__ increments, const uint64_t heads,
                                      const uint64_t frames) {
    const uint64_t total = heads * frames;
    for (uint64_t i = blockIdx.x * static_cast<uint64_t>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<uint64_t>(gridDim.x) * blockDim.x) {
        const uint64_t head = i / frames, frame = i % frames;
        const double ph = __dadd_rn(phases[head], __dmul_rn(increments[head], static_cast<double>(frame)));
        corr[i] = make_float2(static_cast<float>(cos(ph)), static_cast<float>(sin(ph)));
    }
}
__global__ void fir_phase_advance_kernel(double* __restrict__ phases, const double* __restrict__ increments,
                                         const uint64_t heads, const uint64_t frames) {
    const uint64_t head = blockIdx.x * static_cast<uint64_t>(blockDim.x) + threadIdx.x;
    if (head < heads) {
        phases[head] = remainder(__dadd_rn(phases[head], __dmul_rn(increments[head], static_cast<double>(frames))),
                                 2.0 * 3.14159265358979323846);
    }
}

// New history = last L-1 samples of concat(old history, x).
__global__ void fir_history_kernel(const float2* __restrict__ x, const float2* __restrict__ old_hist,
                                   float2* __restrict__ new_hist, const uint64_t n_in, const uint32_t hist_len) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < hist_len; i += gridDim.x * blockDim.x) {
        // element i of the new history is stream index n_in - hist_len + i
        const int64_t j = static_cast<int64_t>(n_in) - hist_len + i;
        new_hist[i] = j >= 0 ? x[j] : old_hist[hist_len + j];
    }
}

}  // namespace b200

using namespace b200;

struct b200_fir_plan {
    b200_ctx* ctx;
    uint32_t L, R, heads;
    bool real_taps;
    bool const_taps = false;
    std::vector<float> taps_host;      // re-ordered table (also uploaded to taps_dev)
    int ob;
    uint32_t lp_pad, hpad, threads, qt, plane_pitch;
    size_t smem;
    // chunk-pair form (fir_decim_kernel<.., PAIR>): real taps, even R, odd L; geometry in 16-byte chunks
    bool pair_ok = false;
    int pair_ob = 0;
    uint32_t pair_lp_pad = 0, pair_hpad = 0, pair_threads = 0, pair_qt = 0, pair_pitch = 0;
    size_t pair_smem = 0;
    std::vector<float> pair_taps_host;  // [heads][R/2][lp_pad] x (h[2c], h[2c-1])
    std::string variant;                // b200_fir_plan_variant
    float* taps_dev;
    float2* hist[2];
    int cur;
    // frequency-translating heads
    bool translate = false;
    uint64_t frame_len = 0;
    float2* rot_dev = nullptr;        // [heads, frame_len / R]
    double* phases_dev = nullptr;     // [heads]
    double* increments_dev = nullptr; // [heads]
    float2* corr_dev = nullptr;       // [heads, corr_frames]
    uint64_t corr_frames = 0;
};

template <int OB, bool REAL_TAPS, bool CONST_TAPS>
static int fir_launch_variant(b200_fir_plan* pl, const FirParams& p, unsigned grid, cudaStream_t s) {
    auto k = fir_decim_kernel<OB, REAL_TAPS, CONST_TAPS>;
    B200_CUDA_CHECK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(pl->smem)));
    k<<<grid, pl->threads, pl->smem, s>>>(p);
    B200_LAUNCH_CHECK();
    return B200_SUCCESS;
}

template <int OB>
static int fir_launch_pair(b200_fir_plan* pl, const FirParams& p, unsigned grid, cudaStream_t s) {
    void (*k)(FirParams) = pl->real_taps ? fir_decim_kernel<OB, true, true, true> : fir_decim_kernel<OB, false, true, true>;
    B200_CUDA_CHECK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(pl->pair_smem)));
    k<<<grid, pl->pair_threads, pl->pair_smem, s>>>(p);
    B200_LAUNCH_CHECK();
    return B200_SUCCESS;
}

// Tile geometry for a stream of `elem_bytes` elements decimated by R with L taps of `tap_floats` floats each: the largest
// odd OB (register sliding window) whose staged planes fit the shared-memory budget.
struct FirGeometry {
    bool ok = false;
    int ob = 0;
    uint32_t threads = 0, lp_pad = 0, hpad = 0, qt = 0, pitch = 0;
    size_t smem = 0;
};
static FirGeometry fir_geometry(const uint32_t L, const uint32_t R, const uint32_t heads, const uint32_t tap_floats,
                                const uint32_t elem_bytes, const int max_ob) {
    FirGeometry g;
    const uint32_t lp = (L + R - 1) / R;
    const int ob_options[4] = {7, 5, 3, 1};
    uint32_t thread_options[3] = {128, 64, 32};
    if (const char* env = getenv("B200_FIR_THREADS")) {          // A/B aid: preferred CTA size
        const int v = atoi(env);
        if (v == 32 || v == 64 || v == 128) {
            thread_options[0] = static_cast<uint32_t>(v);
        }
    }
    const uint32_t period = 128 / elem_bytes;        // elements per 128-byte bank period
    int largest = max_ob;
    if (const char* env = getenv("B200_FIR_OB")) {               // A/B aid: largest OB to consider
        largest = atoi(env);
    }
    const int first_ob = largest <= 1 ? 3 : (largest <= 3 ? 2 : (largest <= 5 ? 1 : 0));
    for (int oi = first_ob; oi < 4 && !g.ok; ++oi) {
        for (int ti = 0; ti < 3 && !g.ok; ++ti) {
            const int ob = ob_options[oi];
            const uint32_t threads = thread_options[ti];
            const uint32_t lp_pad = (lp + ob - 1) / ob * ob;
            const uint32_t hpad = lp_pad + 1;                       // rows of history incl. slack for padded taps
            const uint32_t qt = threads * ob;
            // A warp stages 32 consecutive elements = R planes x 32/R rows with one cp.async each; the planes of one
            // conflict group (16 lanes for 8-byte, 8 lanes for 16-byte elements) land on disjoint banks when the pitch is
            // period / R (mod period) for R | period; an odd pitch otherwise. (The compute phase reads one plane at a
            // time with a lane stride of OB elements, OB odd: any pitch is fine.)
            uint32_t pitch = qt + hpad + 1;
            if (R > 1 && period % R == 0) {
                const uint32_t want = period / R;
                pitch += (want + period - pitch % period) % period;
            } else {
                pitch |= 1u;
            }
            const size_t tap_words = static_cast<size_t>(heads) * R * lp_pad * tap_floats;
            const size_t smem = static_cast<size_t>(R) * pitch * elem_bytes + ((tap_words + 1) & ~size_t(1)) * 4 +
                                static_cast<size_t>(qt) * 8;
            // 128-thread CTAs only while at least four of them fit an SM; otherwise smaller CTAs interleave their
            // load and FMA phases better.
            const size_t limit = (threads == 128 && !getenv("B200_FIR_THREADS")) ? 48 * 1024 : 100 * 1024;
            if (smem <= limit) {
                g.ok = true;
                g.ob = ob;
                g.threads = threads;
                g.lp_pad = lp_pad;
                g.hpad = hpad;
                g.qt = qt;
                g.pitch = pitch;
                g.smem = smem;
            }
        }
    }
    return g;
}

// Most CTAs one exec launches for a tile of `smem` bytes: up to eight per SM, as many as share its shared memory.
static uint64_t fir_cta_cap(const b200_fir_plan* pl, const size_t smem) {
    const uint64_t per_sm = std::max<uint64_t>(1, std::min<uint64_t>(8, (220 * 1024) / (smem + 1024)));
    return static_cast<uint64_t>(pl->ctx->sms) * per_sm;
}

static std::string fir_form_name(const b200_fir_plan* pl, const char* form, const int ob, const uint32_t threads,
                                 const bool const_taps, const uint32_t qt, const size_t smem) {
    char buf[160];
    snprintf(buf, sizeof(buf), "%s OB=%d threads=%u taps=%s %s qt=%u ctas=%llu", form, ob, threads,
             const_taps ? "const" : "shared", pl->real_taps ? "real" : "complex", qt,
             static_cast<unsigned long long>(fir_cta_cap(pl, smem)));
    return buf;
}

template <int OB>
static int fir_launch(b200_fir_plan* pl, const FirParams& p, unsigned grid, cudaStream_t s) {
    if (pl->const_taps) {
        return pl->real_taps ? fir_launch_variant<OB, true, true>(pl, p, grid, s)
                             : fir_launch_variant<OB, false, true>(pl, p, grid, s);
    }
    return pl->real_taps ? fir_launch_variant<OB, true, false>(pl, p, grid, s)
                         : fir_launch_variant<OB, false, false>(pl, p, grid, s);
}

extern "C" {

// filter_taps — FilterTapsImplNativeCpu::generateCoeffs (src/domains/dsp/filter_taps/module_impl_native_cpu.cc:46-80):
// windowed-sinc x Blackman x upconversion, all in F64 with the same libm the reference uses, rounded to CF32.
// STATIC_OUTPUT module: evaluated once on the host (the reference has no CUDA implementation of it either).
int b200_filter_taps_host(double sample_rate, double bandwidth, const double* center, uint64_t heads, uint64_t taps,
                          b200_cf32* out_host) {
    B200_REQUIRE(center && out_host, "b200_filter_taps_host: null argument");
    B200_REQUIRE(std::isfinite(sample_rate) && sample_rate > 0.0, "[MODULE_FILTER_TAPS] Sample rate must be positive.");
    B200_REQUIRE(std::isfinite(bandwidth) && bandwidth > 0.0 && bandwidth <= sample_rate,
                 "[MODULE_FILTER_TAPS] Bandwidth must be between 0 and sample rate.");
    B200_REQUIRE(taps != 0, "[MODULE_FILTER_TAPS] Number of taps cannot be zero.");
    B200_REQUIRE(taps % 2 == 1, "[MODULE_FILTER_TAPS] Number of taps must be odd (%llu).",
                 static_cast<unsigned long long>(taps));
    B200_REQUIRE(heads >= 1, "[MODULE_FILTER_TAPS] At least one center frequency is required.");
    const double kPi = 3.14159265358979323846;
    const double filterWidth = (bandwidth / sample_rate) / 2.0;
    const std::complex<double> j(0.0, 1.0);
    for (uint64_t c = 0; c < heads; ++c) {
        B200_REQUIRE(std::isfinite(center[c]) && center[c] <= sample_rate / 2.0 && center[c] >= -sample_rate / 2.0,
                     "[MODULE_FILTER_TAPS] Center frequency #%llu is outside +-sampleRate/2.",
                     static_cast<unsigned long long>(c));
        const double filterOffset = center[c] / sample_rate;
        for (uint64_t i = 0; i < taps; ++i) {
            const double fi = static_cast<double>(i);
            const double halfLen = static_cast<double>(taps - 1) / 2.0;
            const double n = fi - halfLen;
            const double sincVal = (n == 0.0) ? (2.0 * filterWidth) : std::sin(2.0 * kPi * filterWidth * n) / (kPi * n);
            const double windowVal = (taps == 1) ? 1.0
                                                 : 0.42 - 0.50 * std::cos(2.0 * kPi * fi / (taps - 1)) +
                                                       0.08 * std::cos(4.0 * kPi * fi / (taps - 1));
            const auto upconvert = std::exp(j * 2.0 * kPi * n * filterOffset);
            const auto result = sincVal * windowVal * upconvert;
            out_host[c * taps + i].re = static_cast<float>(result.real());
            out_host[c * taps + i].im = static_cast<float>(result.imag());
        }
    }
    return B200_SUCCESS;
}

int b200_fir_plan_create(b200_ctx* ctx, const b200_cf32* taps_host, uint64_t ntaps, uint64_t heads,
                         uint64_t decimation, b200_fir_plan** plan) {
    B200_REQUIRE(ctx && taps_host && plan, "b200_fir_plan_create: null argument");
    *plan = nullptr;
    B200_REQUIRE(ntaps >= 1 && ntaps <= 65536, "b200_fir_plan_create: tap count %llu out of range (1..65536)",
                 static_cast<unsigned long long>(ntaps));
    B200_REQUIRE(heads >= 1 && heads <= 1024, "b200_fir_plan_create: heads must be in 1..1024");
    B200_REQUIRE(decimation >= 1 && decimation <= 4096, "b200_fir_plan_create: decimation must be in 1..4096");
    DeviceGuard guard(ctx);
    auto* pl = new b200_fir_plan();
    pl->ctx = ctx;
    pl->L = static_cast<uint32_t>(ntaps);
    pl->R = static_cast<uint32_t>(decimation);
    pl->heads = static_cast<uint32_t>(heads);
    pl->real_taps = true;
    for (uint64_t i = 0; i < ntaps * heads; ++i) {
        pl->real_taps = pl->real_taps && taps_host[i].im == 0.0f;
    }
    const FirGeometry geom = fir_geometry(pl->L, pl->R, pl->heads, pl->real_taps ? 1 : 2, 8, 7);
    const bool found = geom.ok;
    if (found) {
        pl->ob = geom.ob;
        pl->threads = geom.threads;
        pl->lp_pad = geom.lp_pad;
        pl->hpad = geom.hpad;
        pl->qt = geom.qt;
        pl->plane_pitch = geom.pitch;
        pl->smem = geom.smem;
    }
    if (!found) {
        delete pl;
        return fail("b200_fir_plan_create: taps=%llu heads=%llu decimation=%llu does not fit the shared-memory tile",
                    static_cast<unsigned long long>(ntaps), static_cast<unsigned long long>(heads),
                    static_cast<unsigned long long>(decimation));
    }
    // Re-order taps per plane: plane p, slot m <- h[kp0 + m R], kp0 = (R - p) % R; zero beyond L.
    const uint32_t per = pl->real_taps ? 1 : 2;
    std::vector<float> host(static_cast<size_t>(pl->heads) * pl->R * pl->lp_pad * per, 0.0f);
    for (uint32_t h = 0; h < pl->heads; ++h) {
        for (uint32_t pidx = 0; pidx < pl->R; ++pidx) {
            const uint32_t kp0 = (pl->R - pidx) % pl->R;
            for (uint32_t m = 0; m < pl->lp_pad; ++m) {
                const uint64_t k = kp0 + static_cast<uint64_t>(m) * pl->R;
                if (k < pl->L) {
                    const b200_cf32 t = taps_host[static_cast<size_t>(h) * pl->L + k];
                    const size_t idx = ((static_cast<size_t>(h) * pl->R + pidx) * pl->lp_pad + m) * per;
                    host[idx] = t.re;
                    if (!pl->real_taps) {
                        host[idx + 1] = t.im;
                    }
                }
            }
        }
    }
    pl->taps_host = host;
    pl->const_taps = host.size() <= kFirConstTapWords && getenv("B200_FIR_SMEM_TAPS") == nullptr;
    // Chunk-pair form: chunk-taps g[c] = (h[2c], h[2c-1]), c < (L+1)/2, decimation R/2, same plane re-ordering.
    if (pl->const_taps && pl->R % 2 == 0 && pl->L % 2 == 1) {
        const uint32_t C = (pl->L + 1) / 2, R2 = pl->R / 2;
        const uint32_t tf = pl->real_taps ? 2 : 4;          // floats per chunk-tap
        // OB = 5 for chunks: a chunk window element already feeds two lane-wise FMAs per output, and the smaller tile
        // lets four 128-thread CTAs (16 warps) share an SM
        const FirGeometry gp = fir_geometry(C, R2, pl->heads, tf, 16, 5);
        const size_t words = static_cast<size_t>(pl->heads) * R2 * gp.lp_pad * tf;
        if (gp.ok && words <= kFirConstTapWords) {
            std::vector<float> pair(words, 0.0f);
            for (uint32_t h = 0; h < pl->heads; ++h) {
                for (uint32_t pidx = 0; pidx < R2; ++pidx) {
                    const uint32_t kp0 = (R2 - pidx) % R2;
                    for (uint32_t m = 0; m < gp.lp_pad; ++m) {
                        const uint64_t c = kp0 + static_cast<uint64_t>(m) * R2;
                        if (c < C) {
                            const size_t idx = ((static_cast<size_t>(h) * R2 + pidx) * gp.lp_pad + m) * tf;
                            const b200_cf32 ta = taps_host[static_cast<size_t>(h) * pl->L + 2 * c];                    // h[2c]
                            const b200_cf32 tb = c > 0 ? taps_host[static_cast<size_t>(h) * pl->L + 2 * c - 1]       // h[2c-1]
                                                       : b200_cf32{0.0f, 0.0f};
                            if (pl->real_taps) {
                                pair[idx] = ta.re;
                                pair[idx + 1] = tb.re;
                            } else {
                                pair[idx] = ta.re;
                                pair[idx + 1] = ta.im;
                                pair[idx + 2] = tb.re;
                                pair[idx + 3] = tb.im;
                            }
                        }
                    }
                }
            }
            pl->pair_ok = true;
            pl->pair_ob = gp.ob;
            pl->pair_lp_pad = gp.lp_pad;
            pl->pair_hpad = gp.hpad;
            pl->pair_threads = gp.threads;
            pl->pair_qt = gp.qt;
            pl->pair_pitch = gp.pitch;
            pl->pair_smem = gp.smem;
            pl->pair_taps_host = pair;
        }
    }
    pl->variant = fir_form_name(pl, "sample", pl->ob, pl->threads, pl->const_taps, pl->qt, pl->smem);
    if (pl->pair_ok) {
        pl->variant += "; " + fir_form_name(pl, "pair", pl->pair_ob, pl->pair_threads, true, pl->pair_qt, pl->pair_smem);
    }
    void* dev = nullptr;
    if (b200_malloc(ctx, host.size() * sizeof(float), &dev) != B200_SUCCESS) {
        delete pl;
        return B200_ERROR;
    }
    pl->taps_dev = static_cast<float*>(dev);
    cudaError_t e = cudaMemcpy(dev, host.data(), host.size() * sizeof(float), cudaMemcpyHostToDevice);
    const size_t hist_bytes = std::max<size_t>(1, pl->L - 1) * sizeof(float2);
    void* h0 = nullptr;
    void* h1 = nullptr;
    if (e != cudaSuccess || b200_malloc(ctx, hist_bytes, &h0) != B200_SUCCESS ||
        b200_malloc(ctx, hist_bytes, &h1) != B200_SUCCESS) {
        cudaFree(dev);
        cudaFree(h0);
        delete pl;
        return fail("b200_fir_plan_create: device setup failed");
    }
    pl->hist[0] = static_cast<float2*>(h0);
    pl->hist[1] = static_cast<float2*>(h1);
    pl->cur = 0;
    cudaStreamSynchronize(cudaStreamLegacy);   // uploads / zero-fills above ran on the legacy stream: settle them before a non-blocking stream executes
    *plan = pl;
    return B200_SUCCESS;
}

const char* b200_fir_plan_variant(const b200_fir_plan* plan) { return plan ? plan->variant.c_str() : ""; }

int b200_fir_plan_set_translation(b200_fir_plan* plan, uint64_t frame_len, const int64_t* center_bins) {
    B200_REQUIRE(plan && center_bins, "b200_fir_plan_set_translation: null argument");
    B200_REQUIRE(frame_len > 0 && frame_len % plan->R == 0,
                 "b200_fir_plan_set_translation: frame length must be a positive multiple of the decimation");
    DeviceGuard guard(plan->ctx);
    const uint64_t M = frame_len + plan->L - 1;            // the reference's convolutionSize
    const uint64_t frame_out = frame_len / plan->R;
    const double kTwoPi = 2.0 * 3.14159265358979323846;
    std::vector<float2> rot(static_cast<size_t>(plan->heads) * frame_out);
    std::vector<double> inc(plan->heads);
    for (uint32_t h = 0; h < plan->heads; ++h) {
        // resamplerOffsets[head] = (-centerBin) mod M  (src/domains/dsp/filter/block_impl.cc:118-160)
        const int64_t c = center_bins[h];
        const uint64_t offset = static_cast<uint64_t>(((-c % static_cast<int64_t>(M)) + static_cast<int64_t>(M)) %
                                                      static_cast<int64_t>(M));
        // fold: bin j of the folded spectrum sums bins (j + g M/R - offset) mod M  ==  time-domain factor
        // exp(+j 2 pi offset n / M) on the full-rate convolution at n = m R (offset == -c mod M).
        for (uint64_t m = 0; m < frame_out; ++m) {
            const uint64_t k = (offset * ((m * plan->R) % M)) % M;
            const double a = kTwoPi * static_cast<double>(k) / static_cast<double>(M);
            rot[static_cast<size_t>(h) * frame_out + m] = make_float2(static_cast<float>(std::cos(a)),
                                                                     static_cast<float>(std::sin(a)));
        }
        // channelPhaseIncrements[head] = remainder(2 pi offset T / M, 2 pi)   (block_impl.cc:519-527), wrapped again
        // by phase_correction (module_impl_native_cpu.cc:70-75)
        inc[h] = std::remainder(std::remainder(kTwoPi * static_cast<double>(offset) * static_cast<double>(frame_len) /
                                                   static_cast<double>(M), kTwoPi), kTwoPi);
    }
    cudaFree(plan->rot_dev);
    cudaFree(plan->phases_dev);
    cudaFree(plan->increments_dev);
    plan->rot_dev = nullptr;
    plan->phases_dev = nullptr;
    plan->increments_dev = nullptr;
    B200_CUDA_CHECK(cudaMalloc(&plan->rot_dev, rot.size() * sizeof(float2)));
    B200_CUDA_CHECK(cudaMalloc(&plan->phases_dev, plan->heads * sizeof(double)));
    B200_CUDA_CHECK(cudaMalloc(&plan->increments_dev, plan->heads * sizeof(double)));
    B200_CUDA_CHECK(cudaMemcpy(plan->rot_dev, rot.data(), rot.size() * sizeof(float2), cudaMemcpyHostToDevice));
    B200_CUDA_CHECK(cudaMemcpy(plan->increments_dev, inc.data(), inc.size() * sizeof(double), cudaMemcpyHostToDevice));
    B200_CUDA_CHECK(cudaMemset(plan->phases_dev, 0, plan->heads * sizeof(double)));
    B200_CUDA_CHECK(cudaStreamSynchronize(cudaStreamLegacy));
    plan->translate = true;
    plan->frame_len = frame_len;
    return B200_SUCCESS;
}

int b200_fir_reset(b200_fir_plan* plan, b200_stream stream) {
    B200_REQUIRE(plan, "b200_fir_reset: null plan");
    DeviceGuard guard(plan->ctx);
    const size_t hist_bytes = std::max<size_t>(1, plan->L - 1) * sizeof(float2);
    B200_CUDA_CHECK(cudaMemsetAsync(plan->hist[plan->cur], 0, hist_bytes, as_stream(stream)));
    if (plan->translate) {
        B200_CUDA_CHECK(cudaMemsetAsync(plan->phases_dev, 0, plan->heads * sizeof(double), as_stream(stream)));
    }
    return B200_SUCCESS;
}

// Time sharding across GPUs (SURVEY.md §8e): a rank that continues a stream another rank (or an earlier call elsewhere)
// started loads the last taps-1 input samples before its slab — the halo — as the plan's history. `count` < taps-1 pads
// the front with zeros (a stream shorter than the filter); a translating plan also takes the number of FRAMES that
// precede the slab so that its phase_correction phasor continues where the previous shard's would be.
int b200_fir_set_history(b200_fir_plan* plan, const b200_cf32* tail_dev, uint64_t count, uint64_t frames_before,
                         b200_stream stream) {
    B200_REQUIRE(plan, "b200_fir_set_history: null plan");
    const uint64_t hist_len = plan->L - 1;
    B200_REQUIRE(count <= hist_len, "b200_fir_set_history: %llu samples given, the history holds taps - 1 = %llu",
                 static_cast<unsigned long long>(count), static_cast<unsigned long long>(hist_len));
    B200_REQUIRE(count == 0 || tail_dev, "b200_fir_set_history: null buffer");
    DeviceGuard guard(plan->ctx);
    const cudaStream_t s = as_stream(stream);
    float2* const hist = plan->hist[plan->cur];
    if (hist_len > count) {
        B200_CUDA_CHECK(cudaMemsetAsync(hist, 0, (hist_len - count) * sizeof(float2), s));
    }
    if (count > 0) {
        B200_CUDA_CHECK(cudaMemcpyAsync(hist + (hist_len - count), tail_dev, count * sizeof(float2),
                                        cudaMemcpyDeviceToDevice, s));
    }
    if (plan->translate) {
        // phase after `frames_before` frames: remainder(inc * frames, 2 pi) per head, as fir_phase_advance_kernel from 0
        B200_CUDA_CHECK(cudaMemsetAsync(plan->phases_dev, 0, plan->heads * sizeof(double), s));
        if (frames_before > 0) {
            fir_phase_advance_kernel<<<static_cast<unsigned>((plan->heads + 63) / 64), 64, 0, s>>>(
                plan->phases_dev, plan->increments_dev, plan->heads, frames_before);
            B200_LAUNCH_CHECK();
        }
    }
    return B200_SUCCESS;
}

int b200_fir_exec(b200_fir_plan* plan, const b200_cf32* x, b200_cf32* y, uint64_t frames, uint64_t frame_len,
                  b200_stream stream) {
    B200_REQUIRE(plan, "b200_fir_exec: null plan");
    const uint64_t n_in = frames * frame_len;
    if (n_in == 0) {
        return B200_SUCCESS;
    }
    B200_REQUIRE(x && y, "b200_fir_exec: null buffer");
    B200_REQUIRE(frame_len % plan->R == 0, "b200_fir_exec: frame length %llu is not a multiple of the decimation %u",
                 static_cast<unsigned long long>(frame_len), plan->R);
    DeviceGuard guard(plan->ctx);
    FirParams p{};
    p.x = reinterpret_cast<const float2*>(x);
    p.hist = plan->hist[plan->cur];
    p.y = reinterpret_cast<float2*>(y);
    p.taps = plan->taps_dev;
    if (plan->const_taps) {
        std::copy(plan->taps_host.begin(), plan->taps_host.end(), p.taps_c);
    }
    p.n_in = n_in;
    p.n_out = n_in / plan->R;
    p.L = plan->L;
    p.R = plan->R;
    p.heads = plan->heads;
    p.lp_pad = plan->lp_pad;
    p.hpad = plan->hpad;
    p.qt = plan->qt;
    p.plane_pitch = plan->plane_pitch;
    p.lp = (plan->L + plan->R - 1) / plan->R;
    p.lp_thr = plan->L - (p.lp - 1) * plan->R;
    p.frame_out = frame_len / plan->R;
    p.frames = frames;
    const cudaStream_t s0 = as_stream(stream);
    if (plan->translate) {
        B200_REQUIRE(frame_len == plan->frame_len, "b200_fir_exec: frame length %llu differs from the translation plan (%llu)",
                     static_cast<unsigned long long>(frame_len), static_cast<unsigned long long>(plan->frame_len));
        if (plan->corr_frames < frames) {
            cudaFree(plan->corr_dev);
            plan->corr_dev = nullptr;
            B200_CUDA_CHECK(cudaMalloc(&plan->corr_dev, plan->heads * frames * sizeof(float2)));
            plan->corr_frames = frames;
        }
        const uint64_t n = plan->heads * frames;
        fir_frame_corr_kernel<<<static_cast<unsigned>(std::min<uint64_t>((n + 127) / 128, 1024)), 128, 0, s0>>>(
            plan->corr_dev, plan->phases_dev, plan->increments_dev, plan->heads, frames);
        B200_LAUNCH_CHECK();
        fir_phase_advance_kernel<<<static_cast<unsigned>((plan->heads + 63) / 64), 64, 0, s0>>>(
            plan->phases_dev, plan->increments_dev, plan->heads, frames);
        B200_LAUNCH_CHECK();
        p.rot = plan->rot_dev;
        p.corr = plan->corr_dev;
    }
    const cudaStream_t s = as_stream(stream);
    int rc = B200_SUCCESS;
    const char* pair_env = getenv("B200_FIR_PAIR");
    const bool use_pair = plan->pair_ok && n_in % 2 == 0 && (reinterpret_cast<uintptr_t>(x) & 15u) == 0 &&
                          !(pair_env && atoi(pair_env) == 0);
    if (use_pair) {
        // the same launch in 16-byte chunk units (see fir_decim_kernel<.., PAIR>)
        FirParams q = p;
        std::copy(plan->pair_taps_host.begin(), plan->pair_taps_host.end(), q.taps_c);
        q.n_in = n_in / 2;
        q.L = (plan->L + 1) / 2;
        q.R = plan->R / 2;
        q.lp_pad = plan->pair_lp_pad;
        q.hpad = plan->pair_hpad;
        q.qt = plan->pair_qt;
        q.plane_pitch = plan->pair_pitch;
        q.lp = (q.L + q.R - 1) / q.R;
        q.lp_thr = q.L - (q.lp - 1) * q.R;
        const uint64_t tiles = (q.n_out + q.qt - 1) / q.qt;
        const unsigned grid = static_cast<unsigned>(std::min<uint64_t>(tiles, fir_cta_cap(plan, plan->pair_smem)));
        switch (plan->pair_ob) {
            case 7: rc = fir_launch_pair<7>(plan, q, grid, s); break;
            case 5: rc = fir_launch_pair<5>(plan, q, grid, s); break;
            case 3: rc = fir_launch_pair<3>(plan, q, grid, s); break;
            default: rc = fir_launch_pair<1>(plan, q, grid, s); break;
        }
    } else {
        const uint64_t tiles = (p.n_out + p.qt - 1) / p.qt;
        const unsigned grid = static_cast<unsigned>(std::min<uint64_t>(tiles, fir_cta_cap(plan, plan->smem)));
        switch (plan->ob) {
            case 7: rc = fir_launch<7>(plan, p, grid, s); break;
            case 5: rc = fir_launch<5>(plan, p, grid, s); break;
            case 3: rc = fir_launch<3>(plan, p, grid, s); break;
            default: rc = fir_launch<1>(plan, p, grid, s); break;
        }
    }
    if (rc != B200_SUCCESS) {
        return rc;
    }
    if (plan->L > 1) {
        const uint32_t hist_len = plan->L - 1;
        fir_history_kernel<<<(hist_len + 255) / 256, 256, 0, s>>>(p.x, plan->hist[plan->cur], plan->hist[plan->cur ^ 1],
                                                                 n_in, hist_len);
        B200_LAUNCH_CHECK();
        plan->cur ^= 1;
    }
    return B200_SUCCESS;
}

int b200_fir_plan_destroy(b200_fir_plan* plan) {
    if (!plan) {
        return B200_SUCCESS;
    }
    DeviceGuard guard(plan->ctx);
    cudaFree(plan->taps_dev);
    cudaFree(plan->hist[0]);
    cudaFree(plan->hist[1]);
    cudaFree(plan->rot_dev);
    cudaFree(plan->phases_dev);
    cudaFree(plan->increments_dev);
    cudaFree(plan->corr_dev);
    delete plan;
    return B200_SUCCESS;
}

}  // extern "C"
