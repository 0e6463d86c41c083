// The per-cycle stages of the reference's frequency-domain filter wiring that have no other entry point here:
// fold, overlap_add and phase_correction (src/domains/dsp/filter/block_impl.cc:350-582 and
// src/domains/dsp/filter_engine/block_impl.cc wire them between the forward and inverse FFTs). pad and unpad are
// strided copies and run on b200_copy_strided.
//
// All three are HBM-bound streaming kernels over contiguous tensors. fold and overlap_add repeat the reference's
// arithmetic operation by operation and are bit-identical to it; phase_correction differs from it only where CUDA's
// F64 sin / cos and glibc's round to different F32 values.
#include <cmath>

#include "common.cuh"

namespace b200 {

namespace {

constexpr int kThreads = 256;
constexpr uint64_t kMaxGridY = 65535;

inline unsigned grid_x(const b200_ctx* ctx, uint64_t items, uint64_t rows) {
    // Enough CTAs along x to fill the device about eight times over when the rows alone do not.
    const uint64_t needed = (items + kThreads - 1) / kThreads;
    const uint64_t rows_in_flight = rows < kMaxGridY ? rows : kMaxGridY;
    uint64_t want = (static_cast<uint64_t>(ctx->sms) * 8 + rows_in_flight - 1) / rows_in_flight;
    if (want < 1) want = 1;
    return static_cast<unsigned>(needed < want ? (needed ? needed : 1) : want);
}

inline unsigned grid_y(uint64_t rows) { return static_cast<unsigned>(rows < kMaxGridY ? rows : kMaxGridY); }

// ---- fold -------------------------------------------------------------------------------------------------------
// src/domains/dsp/fold/module_impl_native_cpu.cc:102-172. Input [outer, axis, inner], output [outer, size, inner];
// out[r, o, i] = (1/R) sum_{g < R} in[r, (o + g size - offset) mod axis, i], summed in F64 in ascending g.

struct FoldGeometry {
    uint64_t outer, axis, inner, size, groups;
    uint64_t channels, channel_inner;   // channel of output element k: (k / channel_inner) % channels
    uint64_t offset;                    // scalar offset (already reduced mod axis) when offsets == nullptr
};

template <typename T>
__device__ __forceinline__ double2 widen(const T v);
template <>
__device__ __forceinline__ double2 widen<float>(const float v) { return make_double2(static_cast<double>(v), 0.0); }
template <>
__device__ __forceinline__ double2 widen<float2>(const float2 v) {
    return make_double2(static_cast<double>(v.x), static_cast<double>(v.y));
}
template <typename T>
__device__ __forceinline__ T narrow(const double2 v);
template <>
__device__ __forceinline__ float narrow<float>(const double2 v) { return static_cast<float>(v.x); }
template <>
__device__ __forceinline__ float2 narrow<float2>(const double2 v) {
    return make_float2(static_cast<float>(v.x), static_cast<float>(v.y));
}

// grid.y walks the outer rows, grid.x the [size, inner] plane of one output row, output axis innermost in memory
// order, so neighbouring threads load neighbouring input elements.
template <typename T, bool kInnerOne>
__global__ void __launch_bounds__(kThreads) fold_kernel(const T* __restrict__ in, T* __restrict__ out,
                                                         const uint64_t* __restrict__ offsets, const FoldGeometry g) {
    const uint64_t plane = g.size * g.inner;
    const double divisor = static_cast<double>(g.groups);
    for (uint64_t r = blockIdx.y; r < g.outer; r += gridDim.y) {
        const T* row_in = in + r * g.axis * g.inner;
        T* row_out = out + r * plane;
        for (uint64_t j = blockIdx.x * static_cast<uint64_t>(blockDim.x) + threadIdx.x; j < plane;
             j += static_cast<uint64_t>(gridDim.x) * blockDim.x) {
            const uint64_t o = kInnerOne ? j : j / g.inner;
            const uint64_t i = kInnerOne ? 0 : j - o * g.inner;
            uint64_t offset = g.offset;
            if (offsets) {
                offset = offsets[((r * plane + j) / g.channel_inner) % g.channels] % g.axis;
            }
            double2 sum = make_double2(0.0, 0.0);
            uint64_t shifted = o;
            for (uint64_t group = 0; group < g.groups; ++group, shifted += g.size) {
                const uint64_t a = shifted >= offset ? shifted - offset : g.axis - (offset - shifted);
                const double2 v = widen<T>(row_in[a * g.inner + i]);
                sum.x = __dadd_rn(sum.x, v.x);
                sum.y = __dadd_rn(sum.y, v.y);
            }
            row_out[j] = narrow<T>(make_double2(__ddiv_rn(sum.x, divisor), __ddiv_rn(sum.y, divisor)));
        }
    }
}

template <typename T>
int launch_fold(b200_ctx* ctx, const void* in, void* out, const uint64_t* offsets, const FoldGeometry& g,
                cudaStream_t stream) {
    const dim3 grid(grid_x(ctx, g.size * g.inner, g.outer), grid_y(g.outer));
    if (g.inner == 1) {
        fold_kernel<T, true><<<grid, kThreads, 0, stream>>>(static_cast<const T*>(in), static_cast<T*>(out), offsets, g);
    } else {
        fold_kernel<T, false><<<grid, kThreads, 0, stream>>>(static_cast<const T*>(in), static_cast<T*>(out), offsets, g);
    }
    B200_LAUNCH_CHECK();
    return B200_SUCCESS;
}

// ---- overlap_add ------------------------------------------------------------------------------------------------
// src/domains/dsp/overlap_add/module_impl_native_cpu.cc:120-202. buffer/out [outer, buffer_len, inner], overlap
// [outer, overlap_len, inner]; the batch coordinate of overlap element k is (k / batch_stride) % batches.

struct OverlapGeometry {
    uint64_t outer, buffer_len, overlap_len, inner, batches, batch_stride;
};

// out = buffer, plus over the first overlap_len samples of each row the previous batch's overlap (batch > 0) or the
// carried tail (batch 0). Reads `previous` only; overlap_add_store_kernel overwrites it in a later launch.
template <typename T>
__global__ void __launch_bounds__(kThreads) overlap_add_kernel(const T* __restrict__ buffer, const T* __restrict__ overlap,
                                                                const T* __restrict__ previous, T* __restrict__ out,
                                                                const OverlapGeometry g) {
    const uint64_t plane = g.buffer_len * g.inner, overlap_plane = g.overlap_len * g.inner;
    for (uint64_t r = blockIdx.y; r < g.outer; r += gridDim.y) {
        for (uint64_t j = blockIdx.x * static_cast<uint64_t>(blockDim.x) + threadIdx.x; j < plane;
             j += static_cast<uint64_t>(gridDim.x) * blockDim.x) {
            T v = buffer[r * plane + j];
            if (j < overlap_plane) {
                const uint64_t k = r * overlap_plane + j;
                const uint64_t batch_hi = k / g.batch_stride;
                const uint64_t batch = batch_hi % g.batches;
                T add;
                if (batch == 0) {
                    add = previous[(batch_hi / g.batches) * g.batch_stride + (k - batch_hi * g.batch_stride)];
                } else {
                    add = overlap[k - g.batch_stride];
                }
                if constexpr (sizeof(T) == sizeof(float2)) {
                    v = fadd2(v, add);
                } else {
                    v = __fadd_rn(v, add);
                }
            }
            out[r * plane + j] = v;
        }
    }
}

// previous = the last batch of overlap (all of it without a batch axis).
template <typename T>
__global__ void __launch_bounds__(kThreads) overlap_add_store_kernel(const T* __restrict__ overlap,
                                                                      T* __restrict__ previous, const uint64_t count,
                                                                      const OverlapGeometry g) {
    for (uint64_t p = blockIdx.x * static_cast<uint64_t>(blockDim.x) + threadIdx.x; p < count;
         p += static_cast<uint64_t>(gridDim.x) * blockDim.x) {
        const uint64_t hi = p / g.batch_stride;
        previous[p] = overlap[(hi * g.batches + g.batches - 1) * g.batch_stride + (p - hi * g.batch_stride)];
    }
}

template <typename T>
int launch_overlap_add(b200_ctx* ctx, const void* buffer, const void* overlap, void* out, void* previous,
                       const OverlapGeometry& g, cudaStream_t stream) {
    const dim3 grid(grid_x(ctx, g.buffer_len * g.inner, g.outer), grid_y(g.outer));
    overlap_add_kernel<T><<<grid, kThreads, 0, stream>>>(static_cast<const T*>(buffer), static_cast<const T*>(overlap),
                                                         static_cast<const T*>(previous), static_cast<T*>(out), g);
    B200_LAUNCH_CHECK();
    const uint64_t count = g.outer * g.overlap_len * g.inner / g.batches;
    const uint64_t blocks = (count + kThreads - 1) / kThreads;
    const uint64_t cap = static_cast<uint64_t>(ctx->sms) * 8;
    overlap_add_store_kernel<T><<<static_cast<unsigned>(blocks < cap ? blocks : cap), kThreads, 0, stream>>>(
        static_cast<const T*>(overlap), static_cast<T*>(previous), count, g);
    B200_LAUNCH_CHECK();
    return B200_SUCCESS;
}

// ---- phase_correction ---------------------------------------------------------------------------------------------
// src/domains/dsp/phase_correction/module_impl_native_cpu.cc:81-115. Element k of a contiguous CF32 tensor belongs to
// batch (k / batch_inner) % batches and channel (k / channel_inner) % channels, and is multiplied by
// (cos phi, sin phi), phi = phases[channel] + wrapped[channel] * batch in F64. Both coordinates are constant over runs
// of `run` = min(batch_inner, channel_inner) elements: one CTA row per run, one F64 sin / cos per CTA and run.

struct PhaseArgs {
    uint64_t runs, run, batches, batch_inner, channels, channel_inner;
    double phases[B200_PHASE_CORRECTION_MAX_CHANNELS];
    double wrapped[B200_PHASE_CORRECTION_MAX_CHANNELS];
};

__global__ void __launch_bounds__(kThreads) phase_correction_kernel(const float2* __restrict__ in,
                                                                     float2* __restrict__ out, const PhaseArgs a) {
    __shared__ float2 correction;
    for (uint64_t r = blockIdx.y; r < a.runs; r += gridDim.y) {
        const uint64_t first = r * a.run;
        if (threadIdx.x == 0) {
            const uint64_t batch = a.batches == 1 ? 0 : (first / a.batch_inner) % a.batches;
            const uint64_t channel = a.channels == 1 ? 0 : (first / a.channel_inner) % a.channels;
            // phases[c] + wrapped[c] * batch, each step rounded (the reference's host build does not contract it)
            const double phi = __dadd_rn(a.phases[channel], __dmul_rn(a.wrapped[channel], static_cast<double>(batch)));
            correction = make_float2(static_cast<float>(cos(phi)), static_cast<float>(sin(phi)));
        }
        __syncthreads();
        const float2 c = correction;
        for (uint64_t j = blockIdx.x * static_cast<uint64_t>(blockDim.x) + threadIdx.x; j < a.run;
             j += static_cast<uint64_t>(gridDim.x) * blockDim.x) {
            out[first + j] = cmul_exact(in[first + j], c);
        }
        __syncthreads();
    }
}

}  // namespace

}  // namespace b200

using namespace b200;

extern "C" {

int b200_fold(b200_ctx* ctx, const void* in, void* out, int is_complex, uint64_t outer, uint64_t axis, uint64_t inner,
              uint64_t size, uint64_t offset, const uint64_t* channel_offsets, uint64_t channels,
              uint64_t channel_inner, b200_stream stream) {
    B200_REQUIRE(ctx && in && out, "b200_fold: null argument");
    B200_REQUIRE(size > 0 && axis % size == 0, "b200_fold: size (%llu) must divide the axis (%llu)",
                 static_cast<unsigned long long>(size), static_cast<unsigned long long>(axis));
    B200_REQUIRE(!channel_offsets || (channels > 0 && channel_inner > 0),
                 "b200_fold: per-channel offsets need channels and channel_inner");
    if (outer == 0 || inner == 0) {
        return B200_SUCCESS;
    }
    FoldGeometry g{outer, axis, inner, size, axis / size, channels ? channels : 1, channel_inner ? channel_inner : 1,
                   offset % axis};
    DeviceGuard guard(ctx);
    return is_complex ? launch_fold<float2>(ctx, in, out, channel_offsets, g, as_stream(stream))
                      : launch_fold<float>(ctx, in, out, channel_offsets, g, as_stream(stream));
}

int b200_overlap_add(b200_ctx* ctx, const void* buffer, const void* overlap, void* out, void* previous, int is_complex,
                     uint64_t outer, uint64_t buffer_len, uint64_t overlap_len, uint64_t inner, uint64_t batches,
                     uint64_t batch_stride, b200_stream stream) {
    B200_REQUIRE(ctx && buffer && overlap && out && previous, "b200_overlap_add: null argument");
    B200_REQUIRE(overlap_len <= buffer_len, "b200_overlap_add: overlap (%llu) longer than the buffer (%llu)",
                 static_cast<unsigned long long>(overlap_len), static_cast<unsigned long long>(buffer_len));
    if (outer == 0 || inner == 0 || buffer_len == 0) {
        return B200_SUCCESS;
    }
    const uint64_t overlap_total = outer * overlap_len * inner;
    B200_REQUIRE(batches > 0 && batch_stride > 0 && overlap_total % (batches * batch_stride) == 0,
                 "b200_overlap_add: batches x batch_stride must tile the overlap tensor");
    const OverlapGeometry g{outer, buffer_len, overlap_len, inner, batches, batch_stride};
    DeviceGuard guard(ctx);
    return is_complex ? launch_overlap_add<float2>(ctx, buffer, overlap, out, previous, g, as_stream(stream))
                      : launch_overlap_add<float>(ctx, buffer, overlap, out, previous, g, as_stream(stream));
}

int b200_phase_correction(b200_ctx* ctx, const b200_cf32* in, b200_cf32* out, uint64_t count, uint64_t batches,
                          uint64_t batch_inner, uint64_t channels, uint64_t channel_inner, const double* phases,
                          const double* wrapped_increments, b200_stream stream) {
    B200_REQUIRE(ctx && in && out && phases && wrapped_increments, "b200_phase_correction: null argument");
    B200_REQUIRE(channels >= 1 && channels <= B200_PHASE_CORRECTION_MAX_CHANNELS,
                 "b200_phase_correction: %llu channels (1 .. %d supported)", static_cast<unsigned long long>(channels),
                 B200_PHASE_CORRECTION_MAX_CHANNELS);
    B200_REQUIRE(batches >= 1 && batch_inner >= 1 && channel_inner >= 1, "b200_phase_correction: bad geometry");
    if (count == 0) {
        return B200_SUCCESS;
    }
    PhaseArgs a{};
    a.batches = batches;
    a.batch_inner = batch_inner;
    a.channels = channels;
    a.channel_inner = channel_inner;
    a.run = count;
    if (batches > 1 && batch_inner < a.run) a.run = batch_inner;
    if (channels > 1 && channel_inner < a.run) a.run = channel_inner;
    B200_REQUIRE(count % a.run == 0, "b200_phase_correction: batch_inner / channel_inner must divide count");
    a.runs = count / a.run;
    for (uint64_t c = 0; c < channels; ++c) {
        a.phases[c] = phases[c];
        a.wrapped[c] = wrapped_increments[c];
    }
    DeviceGuard guard(ctx);
    const dim3 grid(grid_x(ctx, a.run, a.runs), grid_y(a.runs));
    phase_correction_kernel<<<grid, kThreads, 0, as_stream(stream)>>>(reinterpret_cast<const float2*>(in),
                                                                       reinterpret_cast<float2*>(out), a);
    B200_LAUNCH_CHECK();
    return B200_SUCCESS;
}

}  // extern "C"
