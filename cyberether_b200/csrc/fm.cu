// FM quadrature demodulation — replaces FmImplNativeCpu::computeSubmit
// (src/domains/dsp/fm/module_impl_native_cpu.cc:43-175), narrow mode:
//     d[n] = arg(conj(x[n-1]) * x[n]) * ref,   ref = 1 / (2 pi (100e3 / sampleRate))      (module_impl.cc:108-111)
//     first sample ever -> 0; non-finite x[n] or x[n-1] -> NaN (and the de-emphasis state is not touched)
//     optional one-pole de-emphasis y += alpha (d - y), state carried per lane across frames and cycles.
// Tensor layout [frames, lanes, frame_len]: frames (the batch axis) are consecutive in time, lanes
// (channel axis, e.g. filter heads) are independent. Discriminator and de-emphasis are ONE pass over the data
// (12 B/sample): the recurrence is a scan of affine maps y -> g y + o with a decoupled look-back between tiles, each
// thread replaying its own samples from its carry-in in the reference's operation order.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <mutex>
#include <unordered_map>
#include <vector>

#include "common.cuh"

namespace b200 {

struct FmState {          // one per lane, device resident
    float2 previous;
    float deemphasis;
    int has_previous;
};

__device__ __forceinline__ bool finite2(const float2 v) { return isfinite(v.x) && isfinite(v.y); }

// atan2 for finite arguments: a = min(|x|, |y|) / max(|x|, |y|) in [0, 1], atan(a) = a P(a^2) with a degree-8 minimax P
// (max |error| 1.0e-7 evaluated in F32, i.e. < 2 ulp at pi/4; the fit is tools/atan_fit.py), octant fix-ups, IEEE signs
// for zeros (atan2(+-0, x < 0 or -0) = +-pi). ~25 instructions against ~60 of libdevice's atan2f: the narrow kernel is
// instruction-bound (one atan2 per 12 bytes). The reference's std::arg is
// glibc's correctly rounded atan2f; both sit inside the 1e-5 absolute tolerance of the fm tests by two orders.
__device__ __forceinline__ float atan2_finite(const float y, const float x) {
    const float ax = fabsf(x), ay = fabsf(y);
    const float mx = fmaxf(ax, ay), mn = fminf(ax, ay);
    const float a = mx == 0.0f ? 0.0f : __fdividef(mn, mx);
    const float u = a * a;
    float p = 0.0029035410843789577f;
    p = fmaf(p, u, -0.016282962635159492f);
    p = fmaf(p, u, 0.04303929582238197f);
    p = fmaf(p, u, -0.07533670216798782f);
    p = fmaf(p, u, 0.10654674470424652f);
    p = fmaf(p, u, -0.14207133650779724f);
    p = fmaf(p, u, 0.19993053376674652f);
    p = fmaf(p, u, -0.3333309292793274f);
    p = fmaf(p, u, 1.0f);
    float r = p * a;
    r = ay > ax ? 1.5707963705062866f - r : r;
    r = __float_as_int(x) < 0 ? 3.1415927410125732f - r : r;
    return copysignf(r, y);
}

// std::arg(std::conj(p) * c) * ref with the reference's F32 rounding sequence for the products (no FMA contraction).
__device__ __forceinline__ float discriminate(const float2 p, const float2 c, const float ref) {
    const float re = __fadd_rn(__fmul_rn(p.x, c.x), __fmul_rn(p.y, c.y));
    const float im = __fsub_rn(__fmul_rn(p.x, c.y), __fmul_rn(p.y, c.x));
    return __fmul_rn(atan2_finite(im, re), ref);
}

// ---- narrow mode in ONE pass: discriminator + de-emphasis with a decoupled look-back scan ---------------------
// 12 B/sample (8 read, 4 written) instead of the 24 of discriminator + reduce + carry + apply. A CTA takes tiles of
// 2048 consecutive samples of one row (frame, lane), 8 samples per thread:
//   1. 16-byte loads, d[k] in registers (the reference's rounding sequence + atan2f);
//   2. each thread folds its 8 samples into the affine map y -> g y + o of the recurrence (zero-state response o in
//      the reference's operation order, g = (1-alpha)^#finite, carried as the count #finite), a warp-shuffle +
//      shared-memory scan composes them;
//   3. the tile publishes its aggregate map, warp 0 looks back over the predecessor tiles of the same lane (tiles are
//      numbered time-major, lanes innermost: predecessor = id - lanes) combining aggregates until it meets a tile whose
//      inclusive carry is known, publishes its own carry, and
//   4. every thread replays its 8 samples from its own carry-in — again the reference's operation order.
// Slots carry a launch epoch, so nothing is cleared between launches. The grid never exceeds the number of co-resident
// CTAs (a CTA only ever waits on tiles with smaller ids, which are running or done).
constexpr int kFmTileThreads = 256;
constexpr int kFmPerThread = 8;
constexpr int kFmTile = kFmTileThreads * kFmPerThread;

// Two self-validating 64-bit words per tile (64-bit accesses are single-copy atomic, so no fence is needed):
//   a = (epoch << 2 | state) << 32 | bits(c or y)      state 1: aggregate map published as its count c of finite
//                                                      samples (gain (1 - alpha)^c) and o, 2: carry-out y published
//   b = (epoch << 2 | 1)     << 32 | bits(o)
struct FmScanSlot {
    unsigned long long a, b;
};
__device__ __forceinline__ unsigned long long pack_slot(const uint32_t tag, const float value) {
    return (static_cast<unsigned long long>(tag) << 32) | __float_as_uint(value);
}
__device__ __forceinline__ unsigned long long ld_slot(const unsigned long long* p) {
    return *reinterpret_cast<const volatile unsigned long long*>(p);
}
__device__ __forceinline__ void st_slot(unsigned long long* p, const unsigned long long v) {
    *reinterpret_cast<volatile unsigned long long*>(p) = v;
}

struct FmNarrowParams {
    const float2* x;
    float* out;
    FmState* state;
    FmScanSlot* slots;
    uint64_t frames, lanes, frame_len, tiles_per_row, items;
    float ref, alpha;
    uint32_t epoch;
    uint32_t lookback;      // predecessor tiles of finite samples after which (1 - alpha)^n < 2^-31, clamped to 1..32
    float log2_keep;        // log2(1 - alpha) from F64, at least -1e30: the gain of c finite samples is exp2(c log2_keep)
};

template <bool DEEMPH, bool VEC>
__global__ void __launch_bounds__(kFmTileThreads, DEEMPH ? 6 : 8) fm_narrow_fused_kernel(const FmNarrowParams p) {
    __shared__ float warp_c[kFmTileThreads / 32], warp_o[kFmTileThreads / 32];
    const uint32_t t = threadIdx.x, lane_id = t & 31, warp = t >> 5;
    for (uint64_t id = blockIdx.x; id < p.items; id += gridDim.x) {
        // id = ((frame * tiles_per_row) + tile) * lanes + lane
        const uint64_t lane = id % p.lanes;
        const uint64_t ft = id / p.lanes;
        const uint64_t frame = ft / p.tiles_per_row, tile = ft - frame * p.tiles_per_row;
        const uint64_t row = frame * p.lanes + lane;
        const float2* const xr = p.x + row * p.frame_len;
        float* const outr = p.out + row * p.frame_len;
        const uint64_t s0 = tile * kFmTile + static_cast<uint64_t>(t) * kFmPerThread;

        // ---- 1. samples s0-1 .. s0+7 -----------------------------------------------------------------------
        float2 v[kFmPerThread + 1];
        bool has_prev = true;
        if (s0 < p.frame_len) {
            if (s0 > 0) {
                v[0] = xr[s0 - 1];
            } else if (frame > 0) {
                v[0] = p.x[((frame - 1) * p.lanes + lane) * p.frame_len + p.frame_len - 1];
            } else {
                v[0] = p.state[lane].previous;
                has_prev = p.state[lane].has_previous != 0;
            }
        } else {
            v[0] = make_float2(0.f, 0.f);
        }
        if (VEC && s0 + kFmPerThread <= p.frame_len) {
            const float4* const src = reinterpret_cast<const float4*>(xr + s0);
#pragma unroll
            for (int k = 0; k < kFmPerThread / 2; ++k) {
                const float4 q = __ldcs(src + k);
                v[1 + 2 * k] = make_float2(q.x, q.y);
                v[2 + 2 * k] = make_float2(q.z, q.w);
            }
        } else {
#pragma unroll
            for (int k = 0; k < kFmPerThread; ++k) {
                v[1 + k] = s0 + k < p.frame_len ? xr[s0 + k] : make_float2(0.f, 0.f);
            }
        }
        float d[kFmPerThread];
#pragma unroll
        for (int k = 0; k < kFmPerThread; ++k) {
            if (k == 0 && !has_prev) {
                d[k] = 0.0f;
            } else if (finite2(v[k + 1]) && finite2(v[k])) {
                d[k] = discriminate(v[k], v[k + 1], p.ref);
            } else {
                d[k] = __int_as_float(0x7fc00000);
            }
        }

        float y_start = 0.0f;
        if constexpr (DEEMPH) {
            // ---- 2. this thread's map, then the tile-wide scan of map compositions ---------------------------------
            // A map's gain is (1 - alpha)^c for the c finite samples it covers, and the scans carry c, not the gain:
            // every gain is evaluated once from its count as exp2(c log2(1 - alpha)) with log2(1 - alpha) from F64
            // (relative error ~1e-7 for any c). A product of F32 gains compounds one rounding per factor, and the
            // factors of a steady stream are all the same number, so the errors add up instead of cancelling: the
            // rounding of fl(1 - alpha) (up to 2^-25) taken 2048 times, or of a once-rounded (1 - alpha)^8 taken 256
            // times, is 1e-5 on the gain of a tile at 20 MHz with 75 us, which put the de-emphasised output 25 ulps
            // off, three times the reference's own F32 error. Counts are exact in F32 (< 2^24); a known carry is the
            // constant map of count +inf (gain 0). gain(0) == 1 for every accepted alpha: count 0 is the identity map
            // (the look-back's start, unexamined lanes, a thread's empty prefix), so log2_keep is kept finite even where
            // alpha rounds to 1.0f (narrow rates below ~1.2 kHz), and there gain(c >= 1) == 0 as (1 - alpha)^c is.
            const auto gain = [&p](const float c) { return exp2f(c * p.log2_keep); };
            float o = 0.0f, c = 0.0f;
#pragma unroll
            for (int k = 0; k < kFmPerThread; ++k) {
                if (s0 + k < p.frame_len && isfinite(d[k])) {
                    o = __fadd_rn(o, __fmul_rn(p.alpha, __fsub_rn(d[k], o)));
                    c += 1.0f;
                }
            }
            float sc = c, so = o;                                  // inclusive scan inside the warp
#pragma unroll
            for (int off = 1; off < 32; off <<= 1) {
                const float pc = __shfl_up_sync(0xffffffffu, sc, off);
                const float po = __shfl_up_sync(0xffffffffu, so, off);
                if (lane_id >= static_cast<uint32_t>(off)) {
                    so = fmaf(gain(sc), po, so);                   // later map after earlier map
                    sc += pc;
                }
            }
            __syncthreads();                                       // previous tile's shared values are consumed
            if (lane_id == 31) {
                warp_c[warp] = sc;
                warp_o[warp] = so;
            }
            __syncthreads();
            // exclusive prefix of this thread inside the tile: (warps before) then (lanes before)
            float ec = 0.0f, eo = 0.0f, tc = 0.0f, to = 0.0f;      // (ec, eo): warps before mine; (tc, to): whole tile
#pragma unroll
            for (int w = 0; w < kFmTileThreads / 32; ++w) {
                if (w == static_cast<int>(warp)) {
                    ec = tc;
                    eo = to;
                }
                to = fmaf(gain(warp_c[w]), to, warp_o[w]);
                tc += warp_c[w];
            }
            float lc = __shfl_up_sync(0xffffffffu, sc, 1), lo = __shfl_up_sync(0xffffffffu, so, 1);
            if (lane_id == 0) {
                lc = 0.0f;
                lo = 0.0f;
            }
            const float xg = gain(lc + ec), xo = fmaf(gain(lc), eo, lo);   // map of everything before this thread

            // ---- 3. decoupled look-back by warp 0: 32 predecessors per round, nearest first -----------------------------
            // A predecessor that already knows its carry-out y is the constant map (0, y) and ends the search. So does a
            // vanishing gain: a full tile multiplies the state by (1 - alpha)^2048 (<= 0.26 at the module's maximum sample
            // rate of 20 MHz with 75 us, 4e-48 -> 0 at 250 kHz), so once the composed gain of the tiles looked at is below
            // 2^-31 nothing older can move the carry by half an ulp: normally ONE round over aggregates that the
            // neighbouring tiles publish right after their step 2, instead of waiting for a tile ~600 ids back.
            FmScanSlot* const mine = p.slots + id;
            if (t == 0) {
                st_slot(&mine->b, pack_slot((p.epoch << 2) | 1u, to));
                st_slot(&mine->a, pack_slot((p.epoch << 2) | 1u, tc));
            }
            __syncthreads();                                         // warp_c / warp_o of step 2 consumed by every thread
            if (warp == 0) {
                float ac = 0.0f, ao = 0.0f;                          // map of the tiles looked at so far (nearest applied last)
                // first round: only as many predecessors as a stream of finite samples needs for the gain to vanish
                // (p.lookback, 1 for time constants up to ~95 samples): waiting on 32 neighbours that are all in flight
                // makes every tile as slow as the slowest of them
                uint32_t width = p.lookback;
                for (uint64_t back = 1;; back += width, width = 32) {
                    const uint64_t steps = back + lane_id;
                    float mc, mo;
                    bool is_carry;
                    if (lane_id >= width) {                          // not examined this round: identity
                        is_carry = false;
                        mc = 0.0f;
                        mo = 0.0f;
                    } else if (steps * p.lanes > id) {               // before the lane's first tile: the carried state
                        is_carry = true;
                        mc = __int_as_float(0x7f800000);
                        mo = p.state[lane].deemphasis;
                    } else {
                        const FmScanSlot* const slot = p.slots + (id - steps * p.lanes);
                        unsigned long long a = ld_slot(&slot->a);
                        while (static_cast<uint32_t>(a >> 34) != p.epoch) {
                            a = ld_slot(&slot->a);
                        }
                        is_carry = ((a >> 32) & 3u) == 2u;
                        if (is_carry) {
                            mc = __int_as_float(0x7f800000);
                            mo = __uint_as_float(static_cast<uint32_t>(a));
                        } else {
                            unsigned long long b = ld_slot(&slot->b);
                            while (static_cast<uint32_t>(b >> 34) != p.epoch) {
                                b = ld_slot(&slot->b);
                            }
                            mc = __uint_as_float(static_cast<uint32_t>(a));
                            mo = __uint_as_float(static_cast<uint32_t>(b));
                        }
                    }
                    // warp total, nearest (lowest lane) applied last: cur = cur o (cur of lane + off)
#pragma unroll
                    for (int off = 1; off < 32; off <<= 1) {
                        const float fc = __shfl_down_sync(0xffffffffu, mc, off);
                        const float fo = __shfl_down_sync(0xffffffffu, mo, off);
                        if (lane_id + off < 32) {
                            mo = fmaf(gain(mc), fo, mo);
                            mc += fc;
                        }
                    }
                    const float wc = __shfl_sync(0xffffffffu, mc, 0), wo = __shfl_sync(0xffffffffu, mo, 0);
                    ao = fmaf(gain(ac), wo, ao);
                    ac += wc;
                    if (__any_sync(0xffffffffu, is_carry) || gain(ac) < 4.6566129e-10f) {
                        break;
                    }
                }
                if (lane_id == 0) {
                    warp_o[0] = ao;
                }
            }
            __syncthreads();
            const float ao = warp_o[0];
            const float carry = ao;                                  // composed gain 0 or < 2^-31: a constant map
            if (t == 0) {
                const float y_out = fmaf(gain(tc), carry, to);
                st_slot(&mine->a, pack_slot((p.epoch << 2) | 2u, y_out));
                // (the lane's new state is taken from its last tile's slot by fm_state_update_kernel AFTER this kernel:
                // tiles still looking back may read state[lane].deemphasis until the very end)
            }
            y_start = fmaf(xg, carry, xo);
        }

        // ---- 4. replay / store -----------------------------------------------------------------------------------------
        float r[kFmPerThread];
        float y = y_start;
#pragma unroll
        for (int k = 0; k < kFmPerThread; ++k) {
            r[k] = d[k];
            if constexpr (DEEMPH) {
                if (s0 + k < p.frame_len && isfinite(d[k])) {
                    y = __fadd_rn(y, __fmul_rn(p.alpha, __fsub_rn(d[k], y)));
                    r[k] = y;
                }
            }
        }
        if (VEC && s0 + kFmPerThread <= p.frame_len) {
            float4* const dst = reinterpret_cast<float4*>(outr + s0);
            __stcs(dst, make_float4(r[0], r[1], r[2], r[3]));
            __stcs(dst + 1, make_float4(r[4], r[5], r[6], r[7]));
        } else {
#pragma unroll
            for (int k = 0; k < kFmPerThread; ++k) {
                if (s0 + k < p.frame_len) {
                    outr[s0 + k] = r[k];
                }
            }
        }
    }
}

// =====================================================================================================
// Wideband (stereo) FM — src/domains/dsp/fm/module_impl_native_cpu.cc:130-170.
// Per sample the reference runs, sequentially per lane:
//   NCO pilot phase (F32 running sum with wrap, input independent)
//   4 one-pole filters (pilot I/Q, two cascaded)            -> pilotCos, pilotSin
//   sum  = LP3(notch(d))                                     4 biquads
//   diff = LP3(notch(2 d sin(2 (phase + atan2(pilotCos, pilotSin)))))
//   left/right = sum +- diff, optional one-pole de-emphasis each
// Every stage is a small LINEAR recurrence driven by a pointwise function of earlier stages, so each is
// evaluated as a blocked scan: (1) per chunk, zero-state response at the chunk end; (2) serial carry
// propagation over chunks, state <- A^m state + response (A^C pre-evaluated on the host in F64, A^m by stepping
// for the rare chunk that contains non-finite samples); (3) replay of each chunk from its carry with the
// reference's own operation order (no FMA contraction). Non-finite discriminator samples emit NaN and leave
// every filter state untouched, exactly as the reference's `continue` path.
// =====================================================================================================

struct Biquad {
    float b0, b1, b2, a1, a2;
};

struct FmWideCoeffs {
    float pilot_alpha;
    float pilot_phase_increment;
    float deemphasis_alpha;
    int deemphasis;
    Biquad notch;
    Biquad lowpass[3];
};


// FmImpl::applyBiquad (src/domains/dsp/fm/module_impl.cc:157-164), transposed direct form II, no FMA.
__device__ __forceinline__ float biquad_step(const float x, const Biquad& c, float& z1, float& z2) {
    const float y = __fadd_rn(__fmul_rn(c.b0, x), z1);
    z1 = __fadd_rn(__fsub_rn(__fmul_rn(c.b1, x), __fmul_rn(c.a1, y)), z2);
    z2 = __fsub_rn(__fmul_rn(c.b2, x), __fmul_rn(c.a2, y));
    return y;
}

// state.pilotPhase += inc; if (state.pilotPhase >= 2.0f * JST_PI) state.pilotPhase -= 2.0f * JST_PI;
// JST_PI is a double literal, so the comparison and the subtraction happen in F64 and round back to F32.
// The NCO phase is input independent and identical for every lane, and its F32 recurrence cannot be jumped ahead: one
// thread steps it. The step has no branches and no F64: for every F32 a in [2 pi, 2 pi + 1) the reference's wrap
// (float)((double)a - 2 pi) equals fadd(fsub(a, T), C) with T = 6.2831855f (the smallest F32 >= the F64 value of 2 pi;
// (double)a >= 2 pi <=> a >= T) and C = (float)(T - 2 pi) = 1.7484555e-07f — a - T is exact and the rounding of the sum
// never sits near a tie (checked exhaustively over all 2^21 values). Lane 0 fills a shared-memory batch, the warp flushes
// it with coalesced stores instead of one global store per sample in a branchy loop.
__device__ __forceinline__ float nco_step(const float ph, const float inc) {
    const float a = __fadd_rn(ph, inc);
    const float wrapped = __fadd_rn(__fsub_rn(a, 6.2831854820251465f), 1.7484555314695172e-07f);
    return a >= 6.2831854820251465f ? wrapped : a;
}

__global__ void __launch_bounds__(32) fm_wide_phase_kernel(float* __restrict__ phase, float* __restrict__ phase_state,
                                                                  const uint64_t lane_len, const float inc) {
    constexpr uint32_t kBatch = 2048;
    __shared__ float buf[kBatch];
    float ph = *phase_state;
    for (uint64_t base = 0; base < lane_len; base += kBatch) {
        const uint32_t want = lane_len - base < kBatch ? static_cast<uint32_t>(lane_len - base) : kBatch;
        if (threadIdx.x == 0) {
            uint32_t i = 0;
            for (; i + 8 <= want; i += 8) {
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    buf[i + k] = ph;
                    ph = nco_step(ph, inc);
                }
            }
            for (; i < want; ++i) {
                buf[i] = ph;
                ph = nco_step(ph, inc);
            }
        }
        __syncwarp();
        for (uint32_t i = threadIdx.x; i < want; i += 32) {
            phase[base + i] = buf[i];
        }
        __syncwarp();
    }
    if (threadIdx.x == 0) {
        *phase_state = ph;
    }
}

// The same phase sequence WITHOUT the serial chain. The NCO state is a single F32 and its update is input independent,
// so the whole sequence is one orbit of a map on a finite set: the value right after a wrap is
// fl(fl64(a) - 2 pi) for an F32 a in [2 pi, 2 pi + inc) — at most inc / ulp(2 pi) ~ 1e6 distinct values — hence the
// post-wrap phase must repeat within ~1e6 laps = 2 pi / ulp(2 pi) ~ 1.3e7 samples, whatever the sample rate. The plan
// walks that orbit ONCE on the host with the same three F32 operations (b200_fm_plan_create: a few tens of ms), keeps a
// checkpoint every 4 samples over the transient (`pre` samples) and one period (`cycle` samples), and every call then
// regenerates its slice of the sequence in parallel: sample n folds to orbit position pre + (n - pre) mod cycle, a
// thread loads the checkpoint below it and steps <= 3 + 4 times with nco_step itself. Bit-identical to the serial walk
// (tests/test_gpu_filter_fm.py compares against the reference over cycles; tests/test_index_algebra.py checks the
// orbit bookkeeping on the host).
__global__ void fm_wide_phase_table_kernel(float* __restrict__ phase, const float* __restrict__ checkpoints,
                                           const uint64_t n0, const uint64_t len, const uint64_t pre,
                                           const uint64_t cycle, const float inc) {
    const uint64_t i0 = (blockIdx.x * static_cast<uint64_t>(blockDim.x) + threadIdx.x) * 4;
    if (i0 >= len) {
        return;
    }
    const uint64_t n = n0 + i0;
    const uint64_t m = n < pre ? n : pre + (n - pre) % cycle;
    float ph = checkpoints[m >> 2];
    for (uint32_t r = static_cast<uint32_t>(m & 3); r > 0; --r) {
        ph = nco_step(ph, inc);
    }
    const uint32_t count = len - i0 < 4 ? static_cast<uint32_t>(len - i0) : 4u;
    for (uint32_t k = 0; k < count; ++k) {
        phase[i0 + k] = ph;
        ph = nco_step(ph, inc);
    }
}

// Generic blocked scan over S-state systems. System must provide:
//   static constexpr int S;  __device__ bool step(float* state, uint64_t n, lane, bool replay)  — one sample, reference
//   op order; returns false when the sample is skipped (non-finite discriminator); step_homogeneous(state).
//
// Every sample is an affine map of the state, state <- A state + u(n) (A constant per system), and a skipped sample is
// the identity, so a run of samples is the pair (m, b): m = number of applied samples, b = its zero-state response, and
// the state after it is A^m state + b. Pairs compose as (m2, b2) o (m1, b1) = (m1 + m2, A^m2 b1 + b2); A^m is applied
// from a table of A^(2^k) (F64 on the host, rounded to F32) by the binary digits of m — one matrix-vector product for
// the regular power-of-two run lengths, a few for runs shortened by non-finite samples.
//   scan_tile_kernel    a thread steps kScanC samples from zero state (reference op order), the CTA scans the 256 pairs
//                       of its tile (warp Kogge-Stone by shuffles, then across the 8 warps), stores every thread's
//                       exclusive in-tile prefix and the tile aggregate;
//   scan_tiles_kernel   one warp per lane composes the tile aggregates 32 at a time into per-tile carry-in states and the
//                       lane's carry-out for the next call;
//   scan_replay_kernel  thread carry-in = A^m_prefix tile_carry + b_prefix, then the kScanC samples are replayed with the
//                       reference's own operation order and the outputs written.
constexpr int kScanC = 16;
constexpr int kScanThreads = 256;
constexpr int kScanTile = kScanC * kScanThreads;      // 4096 samples
constexpr int kPowBits = 40;                          // A^(2^k), k < 40: runs up to 2^40 samples

// v <- A^m v with the table pw[k][S*S] (row-major) in shared or global memory
template <int S>
__device__ __forceinline__ void apply_power(const float* __restrict__ pw, uint64_t m, float (&v)[S]) {
    for (int k = 0; m != 0 && k < kPowBits; ++k, m >>= 1) {
        if (m & 1) {
            const float* a = pw + k * S * S;
            float r[S];
#pragma unroll
            for (int i = 0; i < S; ++i) {
                float acc = 0.0f;
#pragma unroll
                for (int j = 0; j < S; ++j) {
                    acc = fmaf(a[i * S + j], v[j], acc);
                }
                r[i] = acc;
            }
#pragma unroll
            for (int i = 0; i < S; ++i) {
                v[i] = r[i];
            }
        }
    }
}

// Inclusive scan of (m, b) pairs over the lanes of a warp, lane 0 = earliest samples.
template <int S>
__device__ __forceinline__ void warp_scan_pairs(const float* __restrict__ pw, uint64_t& m, float (&b)[S]) {
    const uint32_t lid = threadIdx.x & 31;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
        const uint64_t m_left = __shfl_up_sync(0xffffffffu, m, off);
        float left[S];
#pragma unroll
        for (int i = 0; i < S; ++i) {
            left[i] = __shfl_up_sync(0xffffffffu, b[i], off);
        }
        if (lid >= static_cast<uint32_t>(off)) {
            apply_power<S>(pw, m, left);              // A^m_mine * b_left
#pragma unroll
            for (int i = 0; i < S; ++i) {
                b[i] += left[i];
            }
            m += m_left;
        }
    }
}

template <int S>
__device__ __forceinline__ void load_power_table(const float* __restrict__ power, float* pw_smem) {
    for (int i = threadIdx.x; i < kPowBits * S * S; i += blockDim.x) {
        pw_smem[i] = power[i];
    }
    __syncthreads();
}

// tile t covers samples [chunk * kScanTile, +kScanTile) of lane; tiles are numbered lane-major: t = lane * tiles_per_lane + chunk
template <class System>
__global__ void __launch_bounds__(kScanThreads) scan_tile_kernel(const System sys, const float* __restrict__ power,
                                                                  float* __restrict__ thread_prefix,   // [threads][S + 1]
                                                                  float* __restrict__ tile_agg,        // [tiles][S + 1]
                                                                  const uint64_t lanes, const uint64_t lane_len,
                                                                  const uint64_t tiles_per_lane) {
    constexpr int S = System::S;
    __shared__ float pw[kPowBits * S * S];
    __shared__ float warp_b[kScanThreads / 32][S];
    __shared__ uint64_t warp_m[kScanThreads / 32];
    load_power_table<S>(power, pw);
    const uint64_t tiles = lanes * tiles_per_lane;
    for (uint64_t tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const uint64_t lane = tile / tiles_per_lane, chunk = tile - lane * tiles_per_lane;
        const uint64_t n0 = chunk * kScanTile + static_cast<uint64_t>(threadIdx.x) * kScanC;
        float st[S];
#pragma unroll
        for (int i = 0; i < S; ++i) {
            st[i] = 0.0f;
        }
        uint64_t m = 0;
        for (uint64_t n = n0; n < n0 + kScanC && n < lane_len; ++n) {
            m += sys.step(st, n, lane, false) ? 1 : 0;
        }
        // inclusive scan inside the warp, then across the warps of the CTA
        warp_scan_pairs<S>(pw, m, st);
        const uint32_t wid = threadIdx.x >> 5, lid = threadIdx.x & 31;
        if (lid == 31) {
            warp_m[wid] = m;
#pragma unroll
            for (int i = 0; i < S; ++i) {
                warp_b[wid][i] = st[i];
            }
        }
        __syncthreads();
        // exclusive prefix of this thread = (pairs of the earlier warps) then (inclusive of the lane to the left)
        uint64_t pm = 0;
        float pb[S];
#pragma unroll
        for (int i = 0; i < S; ++i) {
            pb[i] = 0.0f;
        }
        for (uint32_t w = 0; w < wid; ++w) {         // <= 7 compositions: (warp w) after (prefix so far)
            apply_power<S>(pw, warp_m[w], pb);
#pragma unroll
            for (int i = 0; i < S; ++i) {
                pb[i] += warp_b[w][i];
            }
            pm += warp_m[w];
        }
        const uint64_t m_left = __shfl_up_sync(0xffffffffu, m, 1);
        float left[S];
#pragma unroll
        for (int i = 0; i < S; ++i) {
            left[i] = __shfl_up_sync(0xffffffffu, st[i], 1);
        }
        if (lid != 0) {                               // (inclusive of the left lane) after (earlier warps)
            apply_power<S>(pw, m_left, pb);
#pragma unroll
            for (int i = 0; i < S; ++i) {
                pb[i] += left[i];
            }
            pm += m_left;
        }
        float* const dst = thread_prefix + (tile * kScanThreads + threadIdx.x) * (S + 1);
        dst[0] = __uint_as_float(static_cast<uint32_t>(pm));        // < kScanTile
#pragma unroll
        for (int i = 0; i < S; ++i) {
            dst[1 + i] = pb[i];
        }
        if (threadIdx.x == kScanThreads - 1) {
            // tile aggregate = (this thread's inclusive warp pair (m, st)) after (the earlier warps)
            float agg[S];
            uint64_t am = 0;
#pragma unroll
            for (int i = 0; i < S; ++i) {
                agg[i] = 0.0f;
            }
            for (uint32_t w = 0; w < wid; ++w) {
                apply_power<S>(pw, warp_m[w], agg);
#pragma unroll
                for (int i = 0; i < S; ++i) {
                    agg[i] += warp_b[w][i];
                }
                am += warp_m[w];
            }
            apply_power<S>(pw, m, agg);
            float* const out = tile_agg + tile * (S + 1);
            out[0] = __uint_as_float(static_cast<uint32_t>(am + m));
#pragma unroll
            for (int i = 0; i < S; ++i) {
                out[1 + i] = agg[i] + st[i];
            }
        }
        __syncthreads();                              // warp_m / warp_b are reused by the next tile
    }
}

// One warp per lane: carry-in of every tile (overwrites the tile's aggregate slot) and the lane's carry-out.
template <class System>
__global__ void __launch_bounds__(32) scan_tiles_kernel(const float* __restrict__ power, float* __restrict__ tile_agg,
                                                        float* __restrict__ lane_state, const uint64_t lanes,
                                                        const uint64_t tiles_per_lane) {
    constexpr int S = System::S;
    __shared__ float pw[kPowBits * S * S];
    load_power_table<S>(power, pw);
    const uint32_t lid = threadIdx.x;
    for (uint64_t lane = blockIdx.x; lane < lanes; lane += gridDim.x) {
        float carry[S];                                // state before the current batch of 32 tiles (uniform across lanes)
#pragma unroll
        for (int i = 0; i < S; ++i) {
            carry[i] = lane_state[lane * S + i];
        }
        float* const base = tile_agg + lane * tiles_per_lane * (S + 1);
        for (uint64_t t0 = 0; t0 < tiles_per_lane; t0 += 32) {
            const uint64_t t = t0 + lid;
            const bool live = t < tiles_per_lane;
            uint64_t m = live ? __float_as_uint(base[t * (S + 1)]) : 0;
            float b[S];
#pragma unroll
            for (int i = 0; i < S; ++i) {
                b[i] = live ? base[t * (S + 1) + 1 + i] : 0.0f;
            }
            warp_scan_pairs<S>(pw, m, b);              // inclusive over the batch
            // state after tile t = A^m_incl carry + b_incl; carry-in of tile t = the state after tile t - 1
            float after[S];
#pragma unroll
            for (int i = 0; i < S; ++i) {
                after[i] = carry[i];
            }
            apply_power<S>(pw, m, after);
#pragma unroll
            for (int i = 0; i < S; ++i) {
                after[i] += b[i];
            }
            float in[S];
#pragma unroll
            for (int i = 0; i < S; ++i) {
                const float prev = __shfl_up_sync(0xffffffffu, after[i], 1);
                in[i] = lid == 0 ? carry[i] : prev;
            }
            if (live) {
#pragma unroll
                for (int i = 0; i < S; ++i) {
                    base[t * (S + 1) + 1 + i] = in[i];
                }
            }
            const uint32_t last = static_cast<uint32_t>(tiles_per_lane - t0 < 32 ? tiles_per_lane - t0 : 32) - 1;
#pragma unroll
            for (int i = 0; i < S; ++i) {
                carry[i] = __shfl_sync(0xffffffffu, after[i], last);
            }
        }
        if (lid == 0) {
#pragma unroll
            for (int i = 0; i < S; ++i) {
                lane_state[lane * S + i] = carry[i];
            }
        }
    }
}

template <class System>
__global__ void __launch_bounds__(kScanThreads) scan_replay_kernel(const System sys, const float* __restrict__ power,
                                                                    const float* __restrict__ thread_prefix,
                                                                    const float* __restrict__ tile_carry,
                                                                    const uint64_t lanes, const uint64_t lane_len,
                                                                    const uint64_t tiles_per_lane) {
    constexpr int S = System::S;
    __shared__ float pw[kPowBits * S * S];
    load_power_table<S>(power, pw);
    const uint64_t tiles = lanes * tiles_per_lane;
    for (uint64_t tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const uint64_t lane = tile / tiles_per_lane, chunk = tile - lane * tiles_per_lane;
        const uint64_t n0 = chunk * kScanTile + static_cast<uint64_t>(threadIdx.x) * kScanC;
        const float* const pre = thread_prefix + (tile * kScanThreads + threadIdx.x) * (S + 1);
        float st[S];
#pragma unroll
        for (int i = 0; i < S; ++i) {
            st[i] = tile_carry[tile * (S + 1) + 1 + i];
        }
        apply_power<S>(pw, __float_as_uint(pre[0]), st);
#pragma unroll
        for (int i = 0; i < S; ++i) {
            st[i] += pre[1 + i];
        }
        for (uint64_t n = n0; n < n0 + kScanC && n < lane_len; ++n) {
            sys.step(st, n, lane, true);
        }
    }
}

// Addressing of sample n of `lane` inside [frames, lanes, frame_len].
struct LaneIndex {
    uint64_t lanes, frame_len;
    __device__ __forceinline__ uint64_t operator()(const uint64_t lane, const uint64_t n) const {
        const uint64_t frame = n / frame_len, s = n - frame * frame_len;
        return (frame * lanes + lane) * frame_len + s;
    }
};

// (P) pilot recovery: state [cosStage, sinStage, pilotCos, pilotSin]; replay writes the difference-channel input
//     2 d sin(2 (phase + atan2(pilotCos, pilotSin))) computed from the state BEFORE... no: AFTER this sample's update,
//     as the reference does (module_impl_native_cpu.cc:133-147).
struct PilotSystem {
    static constexpr int S = 4;
    const float* d;         // discriminator output [frames, lanes, frame_len]
    const float* phase;     // [lane_len]
    float* diff_in;         // [frames, lanes, frame_len]
    LaneIndex at;
    float alpha;
    __device__ __forceinline__ bool step(float* st, const uint64_t n, const uint64_t lane, const bool replay) const {
        const uint64_t e = at(lane, n);
        const float v = d[e];
        if (!isfinite(v)) {
            if (replay) {
                diff_in[e] = v;
            }
            return false;
        }
        const float ph = phase[n];
        const float pc = cosf(ph), ps = sinf(ph);
        st[0] = __fadd_rn(st[0], __fmul_rn(alpha, __fsub_rn(__fmul_rn(v, pc), st[0])));
        st[1] = __fadd_rn(st[1], __fmul_rn(alpha, __fsub_rn(__fmul_rn(v, ps), st[1])));
        st[2] = __fadd_rn(st[2], __fmul_rn(alpha, __fsub_rn(st[0], st[2])));
        st[3] = __fadd_rn(st[3], __fmul_rn(alpha, __fsub_rn(st[1], st[3])));
        if (replay) {
            const float offset = atan2f(st[2], st[3]);
            const float carrier = sinf(__fmul_rn(2.0f, __fadd_rn(ph, offset)));
            diff_in[e] = __fmul_rn(__fmul_rn(2.0f, v), carrier);
        }
        return true;
    }
    __device__ __forceinline__ void step_homogeneous(float* st) const {
        st[0] = __fadd_rn(st[0], __fmul_rn(alpha, __fsub_rn(0.0f, st[0])));
        st[1] = __fadd_rn(st[1], __fmul_rn(alpha, __fsub_rn(0.0f, st[1])));
        st[2] = __fadd_rn(st[2], __fmul_rn(alpha, __fsub_rn(st[0], st[2])));
        st[3] = __fadd_rn(st[3], __fmul_rn(alpha, __fsub_rn(st[1], st[3])));
    }
};

// (A) audio path: notch + 3 low-pass biquads; "lanes" here are 2 * lanes: even = sum path (input d), odd =
//     difference path (input diff_in). State [notch z1,z2, lp0 z1,z2, lp1 z1,z2, lp2 z1,z2]. Replay writes in place.
struct AudioSystem {
    static constexpr int S = 8;
    float* sum;             // in: d, out: sum          [frames, lanes, frame_len]
    float* diff;            // in: diff_in, out: difference
    LaneIndex at;
    Biquad notch;
    Biquad lp[3];
    __device__ __forceinline__ float filter(float x, float* st) const {
        x = biquad_step(x, notch, st[0], st[1]);
        x = biquad_step(x, lp[0], st[2], st[3]);
        x = biquad_step(x, lp[1], st[4], st[5]);
        return biquad_step(x, lp[2], st[6], st[7]);
    }
    __device__ __forceinline__ bool step(float* st, const uint64_t n, const uint64_t vlane, const bool replay) const {
        float* const buf = (vlane & 1) ? diff : sum;
        const uint64_t e = at(vlane >> 1, n);
        const float v = buf[e];
        if (!isfinite(v)) {
            return false;
        }
        const float y = filter(v, st);
        if (replay) {
            buf[e] = y;
        }
        return true;
    }
    __device__ __forceinline__ void step_homogeneous(float* st) const { (void)filter(0.0f, st); }
};

// (E) left/right + de-emphasis: state [leftDeemphasis, rightDeemphasis]; writes the interleaved [.., 2] output.
struct StereoSystem {
    static constexpr int S = 2;
    const float* sum;
    const float* diff;
    float* out;             // [frames, lanes, frame_len, 2]
    LaneIndex at;
    float alpha;
    int deemphasis;
    __device__ __forceinline__ bool step(float* st, const uint64_t n, const uint64_t lane, const bool replay) const {
        const uint64_t e = at(lane, n);
        const float s = sum[e], df = diff[e];
        if (!isfinite(s) || !isfinite(df)) {
            if (replay) {
                const float q = __int_as_float(0x7fc00000);
                out[2 * e] = q;
                out[2 * e + 1] = q;
            }
            return false;
        }
        float left = __fadd_rn(s, df), right = __fsub_rn(s, df);
        if (deemphasis) {
            st[0] = __fadd_rn(st[0], __fmul_rn(alpha, __fsub_rn(left, st[0])));
            st[1] = __fadd_rn(st[1], __fmul_rn(alpha, __fsub_rn(right, st[1])));
            left = st[0];
            right = st[1];
        }
        if (replay) {
            out[2 * e] = left;
            out[2 * e + 1] = right;
        }
        return true;
    }
    __device__ __forceinline__ void step_homogeneous(float* st) const {
        if (deemphasis) {
            st[0] = __fadd_rn(st[0], __fmul_rn(alpha, __fsub_rn(0.0f, st[0])));
            st[1] = __fadd_rn(st[1], __fmul_rn(alpha, __fsub_rn(0.0f, st[1])));
        }
    }
};

__global__ void fm_state_update_kernel(const float2* __restrict__ x, FmState* __restrict__ state,
                                       const uint64_t frames, const uint64_t lanes, const uint64_t frame_len,
                                       const FmScanSlot* __restrict__ last_tiles) {
    const uint64_t lane = blockIdx.x * static_cast<uint64_t>(blockDim.x) + threadIdx.x;
    if (lane < lanes) {
        state[lane].previous = x[((frames - 1) * lanes + lane) * frame_len + frame_len - 1];
        state[lane].has_previous = 1;
        if (last_tiles != nullptr) {          // one-pass narrow kernel: carry-out of the lane's last tile
            state[lane].deemphasis = __uint_as_float(static_cast<uint32_t>(last_tiles[lane].a));
        }
    }
}

}  // namespace b200

using namespace b200;

struct b200_fm_plan {
    b200_ctx* ctx;
    uint64_t lanes;
    float ref;
    float alpha;          // 1.0 = de-emphasis disabled
    bool deemphasis;
    bool wide;
    FmState* state;
    FmScanSlot* slots = nullptr;          // look-back slots of the fused narrow kernel
    uint64_t slot_capacity = 0;
    uint32_t epoch = 0;
    // wide mode
    FmWideCoeffs wc;
    float* wide_state;        // [phase(1) | pilot lanes*4 | audio 2*lanes*8 | stereo lanes*2]
    float* power;             // A^(2^k), k < kPowBits: [pilot kPowBits x 16 | audio kPowBits x 64 | stereo kPowBits x 4]
    float* scratch;           // [sum total | diff total | phase lane_len | thread prefixes | tile aggregates]
    uint64_t scratch_total, scratch_lane_len;
    // pilot NCO orbit (fm_wide_phase_table_kernel): checkpoints every 4 samples over transient + one period
    float* nco_checkpoints = nullptr;
    uint64_t nco_pre = 0, nco_cycle = 0;   // cycle == 0: no period found within the cap -> serial kernel
    uint64_t nco_samples = 0;              // samples demodulated since the last reset (host-side, in submission order)
};

namespace {

// Host twin of nco_step (same three IEEE F32 operations; volatile keeps every intermediate in F32).
float nco_step_host(const float ph, const float inc) {
    volatile float a = ph + inc;
    if (a >= 6.2831854820251465f) {
        volatile float d = a - 6.2831854820251465f;
        volatile float w = d + 1.7484555314695172e-07f;
        return w;
    }
    return a;
}

// Walks the NCO orbit from phase 0 until a post-wrap phase repeats. checkpoints[j] = phase of sample 4 j.
bool walk_nco_orbit_uncached(const float inc, std::vector<float>* checkpoints, uint64_t* pre, uint64_t* cycle);

// One walk (0.05 - 0.25 s) per phase increment and process: plans of the same sample rate share it.
bool walk_nco_orbit(const float inc, std::vector<float>* checkpoints, uint64_t* pre, uint64_t* cycle) {
    struct Orbit {
        bool found;
        std::vector<float> checkpoints;
        uint64_t pre, cycle;
    };
    static std::mutex mutex;
    static std::unordered_map<uint32_t, Orbit> cache;
    uint32_t key;
    memcpy(&key, &inc, sizeof(key));
    std::lock_guard<std::mutex> guard(mutex);
    auto it = cache.find(key);
    if (it == cache.end()) {
        Orbit orbit{};
        orbit.found = walk_nco_orbit_uncached(inc, &orbit.checkpoints, &orbit.pre, &orbit.cycle);
        it = cache.emplace(key, std::move(orbit)).first;
    }
    *checkpoints = it->second.checkpoints;
    *pre = it->second.pre;
    *cycle = it->second.cycle;
    return it->second.found;
}

bool walk_nco_orbit_uncached(const float inc, std::vector<float>* checkpoints, uint64_t* pre, uint64_t* cycle) {
    constexpr uint64_t kCap = 1ull << 25;          // > 2 pi / ulp(2 pi) = 1.3e7 samples: the repeat must come earlier
    std::unordered_map<uint32_t, uint64_t> seen;
    seen.reserve(1u << 21);
    checkpoints->clear();
    float ph = 0.0f;
    uint32_t bits;
    memcpy(&bits, &ph, sizeof(bits));
    seen.emplace(bits, 0);
    bool found = false;
    uint64_t n = 0;
    for (; n < kCap; ++n) {
        if ((n & 3) == 0) {
            checkpoints->push_back(ph);
        }
        const float next = nco_step_host(ph, inc);
        if (next < ph) {                             // wrapped: `next` starts a lap
            memcpy(&bits, &next, sizeof(bits));
            const auto it = seen.find(bits);
            if (it != seen.end()) {
                *pre = it->second;
                *cycle = n + 1 - it->second;
                found = true;
                ph = next;
                ++n;
                break;
            }
            seen.emplace(bits, n + 1);
        }
        ph = next;
    }
    if (!found) {
        return false;
    }
    for (int extra = 0; extra < 8; ++extra, ++n) {   // the checkpoint at and just past pre + cycle
        if ((n & 3) == 0) {
            checkpoints->push_back(ph);
        }
        ph = nco_step_host(ph, inc);
    }
    return true;
}

// A^(2^k), k < kPowBits, of a linear update: the one-step matrix from unit vectors stepped through `homogeneous` in
// F64, then repeated squaring in F64; each power rounded to F32 ([k][S*S], row-major).
template <int S, class Fn>
void transition_powers(Fn homogeneous, float* out) {
    double a[S * S];
    for (int j = 0; j < S; ++j) {
        double st[S] = {};
        st[j] = 1.0;
        homogeneous(st);
        for (int i = 0; i < S; ++i) {
            a[i * S + j] = st[i];
        }
    }
    for (int k = 0; k < kPowBits; ++k) {
        for (int i = 0; i < S * S; ++i) {
            out[k * S * S + i] = static_cast<float>(a[i]);
        }
        double sq[S * S];
        for (int i = 0; i < S; ++i) {
            for (int j = 0; j < S; ++j) {
                double acc = 0.0;
                for (int q = 0; q < S; ++q) {
                    acc += a[i * S + q] * a[q * S + j];
                }
                sq[i * S + j] = acc;
            }
        }
        for (int i = 0; i < S * S; ++i) {
            a[i] = sq[i];
        }
    }
}

void biquad_h(const Biquad& c, double& z1, double& z2, double& x) {
    const double y = c.b0 * x + z1;
    z1 = c.b1 * x - c.a1 * y + z2;
    z2 = c.b2 * x - c.a2 * y;
    x = y;
}

}  // namespace

template <class System>
static int run_scan(const System& sys, float* thread_prefix, float* tile_agg, const float* power, float* lane_state,
                    uint64_t lanes, uint64_t lane_len, uint64_t tiles_per_lane, unsigned cap, cudaStream_t s) {
    const uint64_t tiles = lanes * tiles_per_lane;
    const unsigned grid = static_cast<unsigned>(std::min<uint64_t>(tiles, cap));
    scan_tile_kernel<System><<<grid, kScanThreads, 0, s>>>(sys, power, thread_prefix, tile_agg, lanes, lane_len,
                                                          tiles_per_lane);
    B200_LAUNCH_CHECK();
    scan_tiles_kernel<System><<<static_cast<unsigned>(std::min<uint64_t>(lanes, cap)), 32, 0, s>>>(
        power, tile_agg, lane_state, lanes, tiles_per_lane);
    B200_LAUNCH_CHECK();
    scan_replay_kernel<System><<<grid, kScanThreads, 0, s>>>(sys, power, thread_prefix, tile_agg, lanes, lane_len,
                                                            tiles_per_lane);
    B200_LAUNCH_CHECK();
    return B200_SUCCESS;
}

// Pilot NCO phases of samples n0 .. n0 + len - 1 since reset into phase[0 .. len) (orbit-table plans only).
static int launch_nco_phases(const b200_fm_plan* plan, float* phase, uint64_t n0, uint64_t len, cudaStream_t s) {
    const uint64_t quads = (len + 3) / 4;
    fm_wide_phase_table_kernel<<<static_cast<unsigned>((quads + 255) / 256), 256, 0, s>>>(
        phase, plan->nco_checkpoints, n0, len, plan->nco_pre, plan->nco_cycle, plan->wc.pilot_phase_increment);
    B200_LAUNCH_CHECK();
    return B200_SUCCESS;
}

// Launch of the one-pass narrow kernel (discriminator, optional de-emphasis). `out` may be any F32 [frames, lanes, T].
static int launch_narrow_fused(b200_fm_plan* plan, const float2* x, float* out, uint64_t frames, uint64_t frame_len,
                               bool deemph, cudaStream_t s) {
    FmNarrowParams q{};
    q.x = x;
    q.out = out;
    q.state = plan->state;
    q.frames = frames;
    q.lanes = plan->lanes;
    q.frame_len = frame_len;
    q.tiles_per_row = (frame_len + kFmTile - 1) / kFmTile;
    q.items = frames * q.tiles_per_row * plan->lanes;
    q.ref = plan->ref;
    q.alpha = plan->alpha;
    if (deemph) {
        if (plan->slot_capacity < q.items || plan->epoch >= (1u << 29)) {
            cudaFree(plan->slots);
            plan->slots = nullptr;
            plan->slot_capacity = 0;
            B200_CUDA_CHECK(cudaMalloc(&plan->slots, q.items * sizeof(FmScanSlot)));
            B200_CUDA_CHECK(cudaMemsetAsync(plan->slots, 0, q.items * sizeof(FmScanSlot), s));
            plan->slot_capacity = q.items;
            plan->epoch = 0;
        }
        q.slots = plan->slots;
        q.epoch = ++plan->epoch;
        // tiles (of finite samples) until the composed gain (1 - alpha)^n drops below 2^-31
        const double per_tile = static_cast<double>(std::min<uint64_t>(frame_len, kFmTile)) *
                                -std::log1p(-static_cast<double>(plan->alpha));
        const double tiles_needed = per_tile > 0.0 ? std::ceil(21.5 / per_tile) : 32.0;
        q.lookback = static_cast<uint32_t>(std::min(32.0, std::max(1.0, tiles_needed)));
        // alpha == 1.0f gives log2(0) = -inf and 0 * -inf = NaN for the identity map: clamp to a finite -1e30, for
        // which c = 0 still gives exp2(-0) = 1 and c >= 1 gives 0
        q.log2_keep = static_cast<float>(std::max(std::log2(1.0 - static_cast<double>(plan->alpha)), -1e30));
    }
    const bool vec = frame_len % 4 == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0 &&
                     (reinterpret_cast<uintptr_t>(out) & 15) == 0;
    void (*kernel)(FmNarrowParams) =
        deemph ? (vec ? fm_narrow_fused_kernel<true, true> : fm_narrow_fused_kernel<true, false>)
               : (vec ? fm_narrow_fused_kernel<false, true> : fm_narrow_fused_kernel<false, false>);
    int per_sm = 1;
    B200_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kFmTileThreads, 0));
    // every CTA must be resident: a tile only waits on tiles with smaller ids, which then are running or done
    const uint64_t cap = static_cast<uint64_t>(plan->ctx->sms) * static_cast<uint64_t>(per_sm < 1 ? 1 : per_sm);
    kernel<<<static_cast<unsigned>(std::min<uint64_t>(q.items, cap)), kFmTileThreads, 0, s>>>(q);
    B200_LAUNCH_CHECK();
    return B200_SUCCESS;
}

extern "C" {

int b200_fm_plan_create(b200_ctx* ctx, uint64_t lanes, float sample_rate, int wide, int deemphasis_us,
                        b200_fm_plan** plan) {
    B200_REQUIRE(ctx && plan, "b200_fm_plan_create: null argument");
    *plan = nullptr;
    B200_REQUIRE(lanes >= 1, "b200_fm_plan_create: lanes must be positive");
    B200_REQUIRE(std::isfinite(sample_rate) && sample_rate > 0.0f && sample_rate <= 20e6f,
                 "[MODULE_FM] Sample rate must be finite, positive and must not exceed 20 MHz.");
    B200_REQUIRE(deemphasis_us == 0 || deemphasis_us == 50 || deemphasis_us == 75,
                 "[MODULE_FM] De-emphasis must be 'none', '50us', or '75us'.");
    B200_REQUIRE(!wide || sample_rate >= 200e3f,
                 "[MODULE_FM] Wideband mode requires a sample rate of at least 200 kHz.");
    DeviceGuard guard(ctx);
    auto* pl = new b200_fm_plan();
    pl->ctx = ctx;
    pl->lanes = lanes;
    pl->wide = wide != 0;
    // FmImpl::updateCoefficients (src/domains/dsp/fm/module_impl.cc:108-155); F32/F64 mix as written there
    // (JST_PI is a double literal, so `2.0f * JST_PI * x` is evaluated in F64 and rounded on assignment).
    const double kPi = 3.14159265358979323846;
    const float deviation = pl->wide ? 75e3f : 100e3f;
    const float kf = deviation / sample_rate;
    pl->ref = static_cast<float>(1.0f / (2.0f * kPi * kf));
    pl->deemphasis = deemphasis_us != 0;
    const double sr = static_cast<double>(sample_rate);
    if (pl->deemphasis) {
        const double tau = deemphasis_us == 50 ? 50e-6 : 75e-6;
        pl->alpha = static_cast<float>(1.0 - std::exp(-1.0 / (sr * tau)));
    } else {
        pl->alpha = 1.0f;
    }
    void* st = nullptr;
    if (b200_malloc(ctx, lanes * sizeof(FmState), &st) != B200_SUCCESS) {
        delete pl;
        return B200_ERROR;
    }
    pl->state = static_cast<FmState*>(st);
    pl->wide_state = nullptr;
    pl->power = nullptr;
    pl->scratch = nullptr;
    pl->scratch_total = pl->scratch_lane_len = 0;
    if (pl->wide) {
        FmWideCoeffs& w = pl->wc;
        w.pilot_phase_increment = static_cast<float>(2.0f * kPi * 19e3f / sample_rate);
        w.pilot_alpha = static_cast<float>(1.0 - std::exp(-2.0 * kPi * 200.0 / sr));
        w.deemphasis_alpha = pl->alpha;
        w.deemphasis = pl->deemphasis ? 1 : 0;
        const double pilotOmega = 2.0 * kPi * 19e3 / sr;
        const double pilotCosine = std::cos(pilotOmega), pilotSine = std::sin(pilotOmega);
        const double pilotNotchAlpha = pilotSine / (2.0 * 20.0);
        const double pilotNotchA0 = 1.0 + pilotNotchAlpha;
        w.notch.b0 = static_cast<float>(1.0 / pilotNotchA0);
        w.notch.b1 = static_cast<float>(-2.0 * pilotCosine / pilotNotchA0);
        w.notch.b2 = w.notch.b0;
        w.notch.a1 = w.notch.b1;
        w.notch.a2 = static_cast<float>((1.0 - pilotNotchAlpha) / pilotNotchA0);
        const double q[3] = {0.51763809, 0.70710678, 1.93185165};
        const double omega = 2.0 * kPi * 15e3 / sr;
        const double cosine = std::cos(omega), sine = std::sin(omega);
        for (int section = 0; section < 3; ++section) {
            const double alpha = sine / (2.0 * q[section]);
            const double a0 = 1.0 + alpha;
            Biquad& c = w.lowpass[section];
            c.b0 = static_cast<float>((1.0 - cosine) * 0.5 / a0);
            c.b1 = static_cast<float>((1.0 - cosine) / a0);
            c.b2 = c.b0;
            c.a1 = static_cast<float>(-2.0 * cosine / a0);
            c.a2 = static_cast<float>((1.0 - alpha) / a0);
        }
        // Transition matrix powers A^(2^k) of the three systems (F64 -> F32): [pilot 4x4 | audio 8x8 | stereo 2x2] x kPowBits.
        std::vector<float> host_power(static_cast<size_t>(kPowBits) * (16 + 64 + 4));
        const double pa = w.pilot_alpha;
        transition_powers<4>([pa](double* s) {
            s[0] += pa * (0.0 - s[0]);
            s[1] += pa * (0.0 - s[1]);
            s[2] += pa * (s[0] - s[2]);
            s[3] += pa * (s[1] - s[3]);
        }, host_power.data());
        transition_powers<8>([&w](double* s) {
            double x = 0.0;
            biquad_h(w.notch, s[0], s[1], x);
            biquad_h(w.lowpass[0], s[2], s[3], x);
            biquad_h(w.lowpass[1], s[4], s[5], x);
            biquad_h(w.lowpass[2], s[6], s[7], x);
        }, host_power.data() + kPowBits * 16);
        const double da = w.deemphasis ? static_cast<double>(w.deemphasis_alpha) : 0.0;
        transition_powers<2>([da](double* s) {
            s[0] += da * (0.0 - s[0]);
            s[1] += da * (0.0 - s[1]);
        }, host_power.data() + kPowBits * (16 + 64));
        void* dev = nullptr;
        void* wst = nullptr;
        const size_t state_floats = 1 + lanes * 4 + 2 * lanes * 8 + lanes * 2;
        if (b200_malloc(ctx, host_power.size() * sizeof(float), &dev) != B200_SUCCESS ||
            b200_malloc(ctx, state_floats * sizeof(float), &wst) != B200_SUCCESS ||
            cudaMemcpy(dev, host_power.data(), host_power.size() * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess) {
            cudaFree(dev);
            cudaFree(wst);
            cudaFree(pl->state);
            delete pl;
            return fail("b200_fm_plan_create: device setup failed");
        }
        pl->power = static_cast<float*>(dev);
        pl->wide_state = static_cast<float*>(wst);
        std::vector<float> checkpoints;
        uint64_t pre = 0, cycle = 0;
        if (walk_nco_orbit(w.pilot_phase_increment, &checkpoints, &pre, &cycle)) {
            void* cp = nullptr;
            if (b200_malloc(ctx, checkpoints.size() * sizeof(float), &cp) != B200_SUCCESS ||
                cudaMemcpy(cp, checkpoints.data(), checkpoints.size() * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess) {
                cudaFree(cp);
                b200_fm_plan_destroy(pl);
                return fail("b200_fm_plan_create: NCO orbit upload failed");
            }
            pl->nco_checkpoints = static_cast<float*>(cp);
            pl->nco_pre = pre;
            pl->nco_cycle = cycle;
        }
    }
    cudaStreamSynchronize(cudaStreamLegacy);   // uploads / zero-fills above ran on the legacy stream: settle them before a non-blocking stream executes
    *plan = pl;
    return B200_SUCCESS;
}

int b200_fm_reset(b200_fm_plan* plan, b200_stream stream) {
    B200_REQUIRE(plan, "b200_fm_reset: null plan");
    DeviceGuard guard(plan->ctx);
    B200_CUDA_CHECK(cudaMemsetAsync(plan->state, 0, plan->lanes * sizeof(FmState), as_stream(stream)));
    if (plan->wide) {
        const size_t state_floats = 1 + plan->lanes * 4 + 2 * plan->lanes * 8 + plan->lanes * 2;
        B200_CUDA_CHECK(cudaMemsetAsync(plan->wide_state, 0, state_floats * sizeof(float), as_stream(stream)));
        plan->nco_samples = 0;
    }
    return B200_SUCCESS;
}

int b200_fm_exec(b200_fm_plan* plan, const b200_cf32* x, float* out, uint64_t frames, uint64_t frame_len,
                 b200_stream stream) {
    B200_REQUIRE(plan, "b200_fm_exec: null plan");
    const uint64_t total = frames * plan->lanes * frame_len;
    if (total == 0) {
        return B200_SUCCESS;
    }
    B200_REQUIRE(x && out, "b200_fm_exec: null buffer");
    DeviceGuard guard(plan->ctx);
    const cudaStream_t s = as_stream(stream);
    const uint64_t blocks = (total + 255) / 256;
    const uint64_t cap = static_cast<uint64_t>(plan->ctx->sms) * 8;
    const uint64_t lane_len = frames * frame_len;
    (void)blocks;

    if (plan->wide) {
        const uint64_t tiles_per_lane = (lane_len + kScanTile - 1) / kScanTile;
        const uint64_t vlanes = 2 * plan->lanes;
        if (plan->scratch_total < total || plan->scratch_lane_len < lane_len) {
            cudaFree(plan->scratch);
            plan->scratch = nullptr;
            // the widest system (audio: S = 8 over 2 * lanes virtual lanes) sizes the per-thread prefixes and tile slots
            const uint64_t floats = 2 * total + lane_len + vlanes * tiles_per_lane * (kScanThreads + 1) * 9;
            B200_CUDA_CHECK(cudaMalloc(&plan->scratch, floats * sizeof(float)));
            plan->scratch_total = total;
            plan->scratch_lane_len = lane_len;
        }
        float* const sum = plan->scratch;
        float* const diff = sum + total;
        float* const phase = diff + total;
        float* const thread_prefix = phase + lane_len;
        float* const tile_agg = thread_prefix + vlanes * tiles_per_lane * kScanThreads * 9;
        float* const phase_state = plan->wide_state;
        float* const pilot_state = phase_state + 1;
        float* const audio_state = pilot_state + plan->lanes * 4;
        float* const stereo_state = audio_state + vlanes * 8;
        const LaneIndex at{plan->lanes, frame_len};

        if (launch_narrow_fused(plan, reinterpret_cast<const float2*>(x), sum, frames, frame_len, false, s) !=
            B200_SUCCESS) {
            return B200_ERROR;
        }
        if (plan->nco_cycle != 0) {
            if (launch_nco_phases(plan, phase, plan->nco_samples, lane_len, s) != B200_SUCCESS) {
                return B200_ERROR;
            }
        } else {
            fm_wide_phase_kernel<<<1, 32, 0, s>>>(phase, phase_state, lane_len, plan->wc.pilot_phase_increment);
            B200_LAUNCH_CHECK();
        }
        plan->nco_samples += lane_len;
        const unsigned ucap = static_cast<unsigned>(cap);
        PilotSystem pilot{sum, phase, diff, at, plan->wc.pilot_alpha};
        if (run_scan(pilot, thread_prefix, tile_agg, plan->power, pilot_state, plan->lanes, lane_len, tiles_per_lane,
                     ucap, s) != B200_SUCCESS) {
            return B200_ERROR;
        }
        AudioSystem audio{sum, diff, at, plan->wc.notch, {plan->wc.lowpass[0], plan->wc.lowpass[1], plan->wc.lowpass[2]}};
        if (run_scan(audio, thread_prefix, tile_agg, plan->power + kPowBits * 16, audio_state, vlanes, lane_len, tiles_per_lane,
                     ucap, s) != B200_SUCCESS) {
            return B200_ERROR;
        }
        StereoSystem stereo{sum, diff, out, at, plan->wc.deemphasis_alpha, plan->wc.deemphasis};
        if (run_scan(stereo, thread_prefix, tile_agg, plan->power + kPowBits * 80, stereo_state, plan->lanes, lane_len,
                     tiles_per_lane, ucap, s) != B200_SUCCESS) {
            return B200_ERROR;
        }
        fm_state_update_kernel<<<static_cast<unsigned>((plan->lanes + 63) / 64), 64, 0, s>>>(
            reinterpret_cast<const float2*>(x), plan->state, frames, plan->lanes, frame_len, nullptr);
        B200_LAUNCH_CHECK();
        return B200_SUCCESS;
    }

    if (launch_narrow_fused(plan, reinterpret_cast<const float2*>(x), out, frames, frame_len, plan->deemphasis, s) !=
        B200_SUCCESS) {
        return B200_ERROR;
    }
    const FmScanSlot* last_tiles = nullptr;
    if (plan->deemphasis) {
        const uint64_t items = frames * ((frame_len + kFmTile - 1) / kFmTile) * plan->lanes;
        last_tiles = plan->slots + (items - plan->lanes);
    }
    fm_state_update_kernel<<<static_cast<unsigned>((plan->lanes + 63) / 64), 64, 0, s>>>(
        reinterpret_cast<const float2*>(x), plan->state, frames, plan->lanes, frame_len, last_tiles);
    B200_LAUNCH_CHECK();
    return B200_SUCCESS;
}

int b200_fm_plan_destroy(b200_fm_plan* plan) {
    if (!plan) {
        return B200_SUCCESS;
    }
    DeviceGuard guard(plan->ctx);
    cudaFree(plan->state);
    cudaFree(plan->slots);
    cudaFree(plan->wide_state);
    cudaFree(plan->power);
    cudaFree(plan->scratch);
    cudaFree(plan->nco_checkpoints);
    delete plan;
    return B200_SUCCESS;
}

int b200_fm_nco_phases(b200_fm_plan* plan, uint64_t n0, uint64_t len, float* out, b200_stream stream) {
    B200_REQUIRE(plan && plan->wide && plan->nco_cycle != 0, "b200_fm_nco_phases: needs a wideband plan with an NCO orbit");
    if (len == 0) {
        return B200_SUCCESS;
    }
    B200_REQUIRE(out, "b200_fm_nco_phases: null buffer");
    DeviceGuard guard(plan->ctx);
    return launch_nco_phases(plan, out, n0, len, as_stream(stream));
}

/* Host-only twin of the wideband pilot NCO bookkeeping (walk_nco_orbit + the fold of fm_wide_phase_table_kernel): the
 * phases of samples n0 .. n0 + len - 1 since reset, and the orbit's transient / period. For tests and diagnostics. */
int b200_fm_nco_phases_host(float sample_rate, uint64_t n0, uint64_t len, float* out, uint64_t* pre, uint64_t* cycle) {
    B200_REQUIRE(std::isfinite(sample_rate) && sample_rate > 0.0f, "b200_fm_nco_phases_host: bad sample rate");
    const double kPi = 3.14159265358979323846;
    const float inc = static_cast<float>(2.0f * kPi * 19e3f / sample_rate);      // as b200_fm_plan_create
    std::vector<float> checkpoints;
    uint64_t p = 0, c = 0;
    B200_REQUIRE(walk_nco_orbit(inc, &checkpoints, &p, &c), "b200_fm_nco_phases_host: no period within the cap");
    if (pre) {
        *pre = p;
    }
    if (cycle) {
        *cycle = c;
    }
    for (uint64_t i0 = 0; out && i0 < len; i0 += 4) {
        const uint64_t n = n0 + i0;
        const uint64_t m = n < p ? n : p + (n - p) % c;
        float ph = checkpoints[m >> 2];
        for (uint64_t r = m & 3; r > 0; --r) {
            ph = nco_step_host(ph, inc);
        }
        for (uint64_t k = 0; k < 4 && i0 + k < len; ++k) {
            out[i0 + k] = ph;
            ph = nco_step_host(ph, inc);
        }
    }
    return B200_SUCCESS;
}

}  // extern "C"
