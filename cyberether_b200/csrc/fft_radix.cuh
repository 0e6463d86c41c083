// General power-of-two FFT kernel, 16 <= N <= 8192: Stockham autosort with radix-16 passes held in registers
// (16 points per thread per pass; the last pass uses radix N / 16^k as 16/r smaller butterflies), TMA-staged
// input, fused window prologue and C2C / amplitude / amplitude+range epilogue. Same machinery as
// fft4096_kernel (fft4096.cuh) with a generic index scheme:
//
//   pass with sub-transform size Ns and radix r, butterfly j in [0, N/r):   k = j mod Ns
//      u_t = in[j + t N/r] * W_{r Ns}^{k t},  y = DFT_r(u),  out[(j - k) r + k + t Ns] = y_t
//
// A CTA works on a block of THREADS*16 samples = G = BLOCK/N consecutive rows landed by ONE bulk TMA copy into
// a 2-deep ring; passes ping-pong between an exchange buffer X1 and the row's own stage buffer, both addressed
// through pad(a) = a + a/16 (one 8-byte pad per 16 elements), which makes every exchange store conflict-free
// (tests/test_index_algebra.py) — with one __syncthreads per pass boundary. A CTA loops over blocks, and a buffer
// is rewritten only after a barrier that follows its last read: the next block's pass 0 rewrites X1 after a pass or
// R2C unpack barrier, or, for 2 and 4 register passes, after one at the end of the block (a __syncwarp for the
// warp-local rows of 2 passes); the stage buffer is refilled by TMA only after the next block's first barrier.
// Twiddles W^{k t} are thread-constant per (pass, butterfly): stored powers w^1..w^3, w^4, w^8, w^12 from an
// F64-evaluated table.
#pragma once

#include "fft4096.cuh"

namespace b200 {

// ---- radix plan ------------------------------------------------------------------------------
__host__ __device__ constexpr int radix_pass_count(const int log2n) { return (log2n + 3) / 4; }
__host__ __device__ constexpr int radix_of_pass(const int log2n, const int pass) {
    const int done = 4 * pass;
    return log2n - done >= 4 ? 16 : (1 << (log2n - done));
}
__host__ __device__ constexpr int radix_threads(const int log2n) {
    return (1 << log2n) / 16 > 256 ? (1 << log2n) / 16 : 256;
}
__host__ __device__ constexpr int radix_stage_bytes(const int log2n) {
    return (radix_threads(log2n) * 16 + radix_threads(log2n)) * 8;      // BLOCK + BLOCK/16 elements
}
constexpr int kRadixStages = 2;
__host__ __device__ constexpr int radix_smem_bytes(const int log2n) {
    return (kRadixStages + 1) * radix_stage_bytes(log2n) + 64;
}

// ---- small DFTs in registers: result X[k] lands in v[dft_pos<R>(k)] ------------------------------
template <int R>
__host__ __device__ constexpr int dft_pos(const int k) {
    return R == 16 ? 4 * (k & 3) + (k >> 2) : (R == 8 ? 4 * (k & 1) + (k >> 1) : k);
}

__device__ __forceinline__ void dft8(float2* v) {
    constexpr float kH = 0.70710678118654752f;
#pragma unroll
    for (int a0 = 0; a0 < 4; ++a0) {
        bfly2(v[a0], v[a0 + 4]);
    }
    v[5] = cscale(csub_i(v[5], v[5]), kH);      // W8^1
    v[6] = make_float2(v[6].y, -v[6].x);        // W8^2 = -i
    v[7] = cscale(cadd_i(v[7], v[7]), -kH);     // W8^3
    bfly4(v[0], v[1], v[2], v[3]);
    bfly4(v[4], v[5], v[6], v[7]);
}

template <int R>
__device__ __forceinline__ void dft_r(float2* v) {
    if constexpr (R == 16) {
        float2(&a)[16] = *reinterpret_cast<float2(*)[16]>(v);
        dft16(a);
    } else if constexpr (R == 8) {
        dft8(v);
    } else if constexpr (R == 4) {
        bfly4(v[0], v[1], v[2], v[3]);
    } else if constexpr (R == 2) {
        bfly2(v[0], v[1]);
    }
}

// v[dft_pos<R>(t)] *= w^t for the INPUT index t = 1..R-1 (Stockham twiddles multiply the inputs).
template <int R>
__device__ __forceinline__ void twiddle_inputs(float2* v, const TwiddleSet& s) {
#pragma unroll
    for (int t = 1; t < R; ++t) {
        float2 x = v[t];
        if ((t & 3) != 0) {
            x = cmul(x, s.lo[(t & 3) - 1]);
        }
        if ((t >> 2) != 0) {
            x = cmul(x, s.hi[(t >> 2) - 1]);
        }
        v[t] = x;
    }
}

__device__ __forceinline__ uint32_t pad16(const uint32_t a) { return a + (a >> 4); }

// x * W_16^b for a compile-time b in [0, 8) (call sites are fully unrolled).
__device__ __forceinline__ float2 mul_w16(const float2 x, const int b) {
    constexpr float kC = 0.92387953251128674f;  // cos(pi/8)
    constexpr float kS = 0.38268343236508977f;  // sin(pi/8)
    constexpr float kH = 0.70710678118654752f;  // sqrt(1/2)
    switch (b) {
        case 0: return x;
        case 1: return cmul(x, make_float2(kC, -kS));
        case 2: return cscale(csub_i(x, x), kH);
        case 3: return cmul(x, make_float2(kS, -kC));
        case 4: return make_float2(x.y, -x.x);
        case 5: return cmul(x, make_float2(-kS, -kC));
        case 6: return cscale(cadd_i(x, x), -kH);
        default: return cmul(x, make_float2(-kC, -kS));
    }
}

// Powers w^1, w^2, w^3, w^4, w^8, w^12 of w = W_n^base from the table W_n^j (indices wrap mod n; only the powers a
// radix actually uses are consumed, the rest are dead code).
__device__ __forceinline__ TwiddleSet load_twiddles_n(const float2* __restrict__ table, const uint32_t base,
                                                      const uint32_t n) {
    TwiddleSet s;
#pragma unroll
    for (int m = 0; m < 3; ++m) {
        s.lo[m] = table[(base * (m + 1)) & (n - 1)];
        s.hi[m] = table[(base * 4 * (m + 1)) & (n - 1)];
    }
    return s;
}

// X[k] of real row `row` (length 2N): layout 0 = [rows, N + 1] CF32, layout 1 = FFTPACK [Re X0, Re X1, Im X1, ..., Re XN].
template <int N>
__device__ __forceinline__ void real_store(void* out, const int layout, const uint64_t row, const uint32_t k, const float2 x) {
    if (layout == 0) {
        static_cast<float2*>(out)[row * (N + 1) + k] = x;
    } else {
        float* const r = static_cast<float*>(out) + row * (2ull * N);
        if (k == 0) {
            r[0] = x.x;
        } else if (k == N) {
            r[2 * N - 1] = x.x;
        } else {
            r[2 * k - 1] = x.x;
            r[2 * k] = x.y;
        }
    }
}

// One CTA per SM guaranteed: on sm_90 (scalar complex arithmetic) a 128-register cap makes the 256-thread forms spill;
// uncapped they spill nothing and measured no slower at any length on H100 (the n = 1024 chain 6 % faster).
template <int LOG2N, int MODE, int WIN>
__global__ void __launch_bounds__(radix_threads(LOG2N), 1)
    fft_radix_kernel(const FftParams p) {
    constexpr int N = 1 << LOG2N;
    constexpr int THREADS = radix_threads(LOG2N);
    constexpr int BLOCK = THREADS * 16;          // samples per CTA iteration
    constexpr int G = BLOCK / N;                 // rows per CTA iteration
    constexpr int T = N / 16;                    // threads per row
    constexpr int PASSES = radix_pass_count(LOG2N);
    constexpr int STAGE_BYTES = radix_stage_bytes(LOG2N);

    extern __shared__ __align__(128) unsigned char smem_raw[];
    float2* const x1 = reinterpret_cast<float2*>(smem_raw + kRadixStages * STAGE_BYTES);
    uint64_t* const full = reinterpret_cast<uint64_t*>(smem_raw + (kRadixStages + 1) * STAGE_BYTES);

    const uint32_t tid = threadIdx.x;
    const uint32_t g = tid / T, lt = tid % T;
    const uint64_t blocks_total = (p.rows + G - 1) / G;
    const uint64_t first = blockIdx.x, stride = gridDim.x;
    const uint32_t my_blocks =
        first < blocks_total ? static_cast<uint32_t>((blocks_total - first + stride - 1) / stride) : 0u;

    if (tid == 0) {
#pragma unroll
        for (int s = 0; s < kRadixStages; ++s) {
            mbar_init(&full[s], 1);
        }
        fence_mbar_init();
    }
    __syncthreads();

    // bytes of block b (the last block of the batch may hold fewer than G rows)
    auto block_bytes = [&](const uint64_t b) -> uint32_t {
        const uint64_t row0 = b * G;
        const uint64_t rows = p.rows - row0 < G ? p.rows - row0 : G;
        return static_cast<uint32_t>(rows * N * 8);
    };

    uint32_t issued = 0;
    if (tid == 0) {
#pragma unroll
        for (int s = 0; s < kRadixStages; ++s) {
            if (issued < my_blocks) {
                const uint64_t b = first + issued * stride;
                const uint32_t bytes = block_bytes(b);
                mbar_expect_tx(&full[s], bytes);
                tma_load_row(smem_raw + s * STAGE_BYTES, p.in + b * BLOCK, bytes, &full[s]);
                ++issued;
            }
        }
    }

    // Thread-constant twiddles: pass q >= 1, butterfly b: w = W_{r Ns}^{k}, k = (lt + b T) mod Ns.
    // Stored for passes 1 and 2 (radix 16: one butterfly; smaller radix: 16/r butterflies); pass 3 (N = 8192
    // only, radix 2) loads its single twiddle on the fly.
    TwiddleSet tw_a;                                   // pass 1 (Ns = 16), radix r1
    constexpr int R1 = PASSES > 1 ? radix_of_pass(LOG2N, 1) : 1;
    constexpr int C1 = PASSES > 1 ? 16 / R1 : 1;
    TwiddleSet tw_a_multi[C1 > 1 ? C1 : 1];
    if constexpr (PASSES > 1) {
        if constexpr (C1 == 1) {
            const uint32_t k = lt & 15;
            tw_a = load_twiddles_n(p.twiddle, k * (N / (R1 * 16)), N);
        } else {
#pragma unroll
            for (int b = 0; b < C1; ++b) {
                const uint32_t k = (lt + b * T) & 15;
                tw_a_multi[b] = load_twiddles_n(p.twiddle, k * (N / (R1 * 16)), N);
            }
        }
    }
    constexpr int R2 = PASSES > 2 ? radix_of_pass(LOG2N, 2) : 1;
    constexpr int C2 = PASSES > 2 ? 16 / R2 : 1;
    TwiddleSet tw_b[C2];
    if constexpr (PASSES > 2) {
#pragma unroll
        for (int b = 0; b < C2; ++b) {
            const uint32_t k = (lt + b * T) & 255;
            tw_b[b] = load_twiddles_n(p.twiddle, k * (N / (R2 * 256)), N);
        }
    }

    float wr[16];
    if constexpr (WIN == WIN_REAL) {
#pragma unroll
        for (int t = 0; t < 16; ++t) {
            wr[t] = p.win_re[lt + t * T];
        }
    }
    float2 tw_last = make_float2(1.f, 0.f);            // pass 3 (N = 8192): W_N^lt
    if constexpr (PASSES > 3) {
        tw_last = p.twiddle[lt];
    }

    uint32_t stage = 0, parity = 0, refill_stage = 0;
    for (uint32_t i = 0; i < my_blocks; ++i) {
        const uint64_t blk = first + static_cast<uint64_t>(i) * stride;
        const uint64_t row = blk * G + g;
        const bool row_valid = row < p.rows;
        float2* const sbuf = reinterpret_cast<float2*>(smem_raw + stage * STAGE_BYTES);
        mbar_wait(&full[stage], parity);

        float2 v[16];
        // ---- pass 0: radix 16 (or N itself when N == 16), Ns = 1, reads the linear TMA block ---------
        {
#pragma unroll
            for (int t = 0; t < 16; ++t) {
                float2 x = sbuf[g * N + lt + t * T];
                if constexpr (MODE == MODE_C2C) {
                    if (p.inverse) {
                        x = make_float2(x.y, x.x);
                    }
                }
                if constexpr (WIN == WIN_REAL) {
                    x = apply_window<WIN>(x, wr[t], make_float2(0.f, 0.f));
                } else if constexpr (WIN == WIN_COMPLEX) {
                    x = apply_window<WIN>(x, 0.f, p.win_c[lt + t * T]);
                }
                v[t] = x;
            }
            if constexpr (PASSES == 1) {
                // single-pass sizes: the stage buffer is consumed here; refill it for the block two ahead
                __syncthreads();
                if (tid == 0 && issued < my_blocks) {
                    const uint64_t b = first + static_cast<uint64_t>(issued) * stride;
                    const uint32_t bytes = block_bytes(b);
                    fence_proxy_async();
                    mbar_expect_tx(&full[stage], bytes);
                    tma_load_row(smem_raw + stage * STAGE_BYTES, p.in + b * BLOCK, bytes, &full[stage]);
                    ++issued;
                }
            }
            dft16(*reinterpret_cast<float2(*)[16]>(v));
            if constexpr (PASSES > 1) {
#pragma unroll
                for (int t = 0; t < 16; ++t) {
                    x1[pad16(g * N + lt * 16 + t)] = v[dft_pos<16>(t)];       // j0 = 16 j, Ns = 1
                }
            }
        }
        if constexpr (PASSES > 1) {
            __syncthreads();
            // The previous block's stage buffer is free now: refill it.
            if (tid == 0 && i >= 1 && issued < my_blocks) {
                const uint64_t b = first + static_cast<uint64_t>(issued) * stride;
                const uint32_t bytes = block_bytes(b);
                fence_proxy_async();
                mbar_expect_tx(&full[refill_stage], bytes);
                tma_load_row(smem_raw + refill_stage * STAGE_BYTES, p.in + b * BLOCK, bytes, &full[refill_stage]);
                ++issued;
            }
            // ---- pass 1: Ns = 16, reads X1, writes the stage buffer (or the output when it is the last) ---
#pragma unroll
            for (int b = 0; b < C1; ++b) {
                const uint32_t j = lt + b * T;
                const uint32_t k = j & 15;
#pragma unroll
                for (int t = 0; t < R1; ++t) {
                    v[b * R1 + t] = x1[pad16(g * N + j + t * (N / R1))];
                }
                if constexpr (C1 == 1) {
                    twiddle_inputs<R1>(v + b * R1, tw_a);
                } else {
                    twiddle_inputs<R1>(v + b * R1, tw_a_multi[b]);
                }
                dft_r<R1>(v + b * R1);
                if constexpr (PASSES > 2) {
                    const uint32_t j0 = (j - k) * R1 + k;
#pragma unroll
                    for (int t = 0; t < R1; ++t) {
                        sbuf[pad16(g * N + j0 + t * 16)] = v[b * R1 + dft_pos<R1>(t)];
                    }
                }
            }
        }
        if constexpr (PASSES > 2) {
            __syncthreads();
            // ---- pass 2: Ns = 256, reads the stage buffer --------------------------------------------------
#pragma unroll
            for (int b = 0; b < C2; ++b) {
                const uint32_t j = lt + b * T;
                const uint32_t k = j & 255;
#pragma unroll
                for (int t = 0; t < R2; ++t) {
                    v[b * R2 + t] = sbuf[pad16(g * N + j + t * (N / R2))];
                }
                twiddle_inputs<R2>(v + b * R2, tw_b[b]);
                dft_r<R2>(v + b * R2);
                if constexpr (PASSES > 3) {
                    const uint32_t j0 = (j - k) * R2 + k;
#pragma unroll
                    for (int t = 0; t < R2; ++t) {
                        x1[pad16(g * N + j0 + t * 256)] = v[b * R2 + dft_pos<R2>(t)];
                    }
                }
            }
        }
        constexpr int RL = radix_of_pass(LOG2N, PASSES - 1);     // radix of the last pass
        constexpr int CL = 16 / RL;
        if constexpr (PASSES > 3) {
            __syncthreads();
            // ---- pass 3 (N = 8192): radix 2, Ns = 4096, single twiddle W_N^k per butterfly --------------------
            // W_N^j with j = lt + b T and T = N / 16: W_N^lt (thread constant, tw_last) times the compile-time constant
            // W_16^b — no table loads in the row loop (they were the kernel's long-scoreboard stalls).
#pragma unroll
            for (int b = 0; b < CL; ++b) {
                const uint32_t j = lt + b * T;                   // k = j (j < Ns)
                v[b * RL] = x1[pad16(g * N + j)];
                v[b * RL + 1] = mul_w16(cmul(x1[pad16(g * N + j + N / 2)], tw_last), b);
                bfly2(v[b * RL], v[b * RL + 1]);
            }
        }

        // ---- epilogue: the last pass has Ns = N / RL, so k = j and output index = j + t Ns --------------------
        if constexpr (MODE == MODE_R2C) {
            // The row is a REAL row of length 2N (z[m] = x[2m] + i x[2m+1]); with Z = FFT_N(z) in registers,
            //   X[k] = e + w o, X[N-k] = conj(e - w o), e = (Z[k] + conj Z[N-k]) / 2, o = (Z[k] - conj Z[N-k]) / (2i), w = W_2N^k.
            // Z goes through the exchange buffer the last pass did NOT read (linear layout), one thread per mirror pair.
            static_assert(PASSES >= 2, "the fused real unpack needs a free exchange buffer");
            constexpr int NS_LAST = N / RL;
            float2* const zbuf = (PASSES % 2 == 1) ? x1 : sbuf;
#pragma unroll
            for (int b = 0; b < CL; ++b) {
#pragma unroll
                for (int t = 0; t < RL; ++t) {
                    zbuf[g * N + lt + b * T + t * NS_LAST] = v[b * RL + dft_pos<RL>(t)];
                }
            }
            __syncthreads();
            if (row_valid) {
                const float2* const zr = zbuf + g * N;
#pragma unroll
                for (int j = 0; j <= 8; ++j) {
                    const uint32_t k = lt + j * T;
                    if (j == 8 && lt != 0) {
                        break;                                   // k = N / 2 belongs to lt == 0 only
                    }
                    if (k == 0) {
                        const float2 a = zr[0];
                        real_store<N>(p.real_out, p.real_layout, row, 0, make_float2(a.x + a.y, 0.0f));
                        real_store<N>(p.real_out, p.real_layout, row, N, make_float2(a.x - a.y, 0.0f));
                        continue;
                    }
                    const float2 a = zr[k];
                    const float2 m = zr[N - k];
                    const float2 e = make_float2(0.5f * (a.x + m.x), 0.5f * (a.y - m.y));
                    const float2 o = make_float2(0.5f * (a.y + m.y), -0.5f * (a.x - m.x));
                    float sn, cs;
                    sincospif(-static_cast<float>(k) * (1.0f / static_cast<float>(N)), &sn, &cs);
                    const float2 tt = make_float2(cs * o.x - sn * o.y, cs * o.y + sn * o.x);
                    real_store<N>(p.real_out, p.real_layout, row, k, make_float2(e.x + tt.x, e.y + tt.y));
                    if (2 * k != N) {
                        real_store<N>(p.real_out, p.real_layout, row, N - k, make_float2(e.x - tt.x, -(e.y - tt.y)));
                    }
                }
            }
            if constexpr (PASSES % 2 == 1) {
                __syncthreads();      // zbuf = X1: the next block's pass 0 rewrites it before its first barrier
            }
        } else if (row_valid) {
            constexpr int NS_LAST = N / RL;
            if constexpr (MODE == MODE_C2C || MODE == MODE_C2C_T) {
                // MODE_C2C_T: row = 16 * transform + k1, element k2 lands at k1 + 16 k2 of the 16 N-point transform
                constexpr int KS = MODE == MODE_C2C_T ? 16 : 1;
                float2* const out = MODE == MODE_C2C_T ? static_cast<float2*>(p.out) + (row >> 4) * (16ull * N) + (row & 15)
                                                       : static_cast<float2*>(p.out) + row * N;
#pragma unroll
                for (int b = 0; b < CL; ++b) {
#pragma unroll
                    for (int t = 0; t < RL; ++t) {
                        float2 X = v[b * RL + dft_pos<RL>(t)];
                        if (p.inverse) {
                            X = make_float2(X.y, X.x);
                        }
                        stg_stream_f2(out + (lt + b * T + t * NS_LAST) * KS, X);
                    }
                }
            } else {
                float* const out = static_cast<float*>(p.out) + row * N;
#pragma unroll
                for (int e = 0; e < 16; e += 2) {
                    const int b0 = e / RL, t0 = e % RL, b1 = (e + 1) / RL, t1 = (e + 1) % RL;
                    const float2 r = spectral_epilogue2<MODE>(v[b0 * RL + dft_pos<RL>(t0)],
                                                              v[b1 * RL + dft_pos<RL>(t1)], p);
                    stg_stream_f1(out + lt + b0 * T + t0 * NS_LAST, r.x);
                    stg_stream_f1(out + lt + b1 * T + t1 * NS_LAST, r.y);
                }
            }
        }
        // With 2 or 4 passes the last pass read X1 across the row's threads and no barrier has followed (R2C's unpack
        // has one): order those reads before the next block's pass 0 rewrites X1. Rows of 2-pass lengths are warp-local.
        if constexpr (MODE != MODE_R2C && PASSES == 4) {
            __syncthreads();
        }
        if constexpr (MODE != MODE_R2C && PASSES == 2) {
            static_assert(32 % T == 0, "a row of a two-pass length must lie within one warp");
            __syncwarp();
        }

        refill_stage = stage;
        if (++stage == kRadixStages) {
            stage = 0;
            parity ^= 1;
        }
    }
}

}  // namespace b200
