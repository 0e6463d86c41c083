/* libb200dsp — Hopper (sm_90a) compute backend for the Jetstream DSP module compute() path.
 *
 * Pure C ABI: POD arguments only, no C++/torch types. Every entry point
 *   - returns an int that follows the reference's `Result` numbering
 *     (include/jetstream/types.hh:19-30): 0 SUCCESS, 1 ERROR, 3 FATAL;
 *   - never throws, never synchronises the stream it is given (except the *_create/_destroy,
 *     malloc/free and explicit *_synchronize calls), and never touches host copies of tensors;
 *   - leaves ownership of every buffer with the caller (device pointers unless stated).
 * `b200_last_error()` returns the thread-local text of the last failure — the string the
 * reference-side shim forwards to JST_ERROR (include/jetstream/logger.hh).
 *
 * Each function names the reference interface (path:line under the reference tree) whose
 * computeSubmit()/create() work it replaces. The reference-side binding is in INTEGRATION.md.
 */
#ifndef B200DSP_H
#define B200DSP_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200_SUCCESS 0
#define B200_ERROR   1
#define B200_FATAL   3

typedef struct b200_ctx b200_ctx;                 /* one per device (replaces Backend::State<CUDA>) */
typedef struct b200_fft_plan b200_fft_plan;
typedef struct b200_chain_plan b200_chain_plan;
typedef struct b200_fir_plan b200_fir_plan;
typedef struct b200_fm_plan b200_fm_plan;
typedef void* b200_stream;                        /* cudaStream_t; NULL = legacy default stream */
typedef void* b200_event;                         /* cudaEvent_t */
typedef struct { float re, im; } b200_cf32;       /* CF32 = std::complex<float> layout */

/* ---- backend / memory ------------------------------------------------------------------ */

/* Library/ABI identification. */
const char* b200_version(void);
const char* b200_last_error(void);

/* src/backend/devices/cuda/base.cc:9-149 (device discovery, one context per deviceId). */
int b200_device_count(int* count);
int b200_ctx_create(int device, b200_ctx** ctx);
int b200_ctx_destroy(b200_ctx* ctx);
int b200_ctx_device(const b200_ctx* ctx, int* device);
int b200_ctx_sm_count(const b200_ctx* ctx, int* sms);
/* What Backend::CUDA caches about its device at construction (src/backend/devices/cuda/base.cc:46-107: name, compute
 * capability, API version, integrated / discrete, memory, host-memory import capability). */
typedef struct {
    char name[256];
    int device;
    int compute_capability_major, compute_capability_minor;
    int sm_count;
    int integrated;
    int can_map_host_memory;
    int can_use_host_pointer_for_registered_memory;
    int runtime_version;                    /* cudaRuntimeGetVersion: 1000 major + 10 minor */
    uint64_t total_memory_bytes;
    uint64_t shared_memory_per_block_optin;
} b200_device_info;
int b200_ctx_info(const b200_ctx* ctx, b200_device_info* info);

/* src/memory/buffer_cuda.cc:31-124 (device allocation, zero-filled like cudaMemset at :119). */
int b200_malloc(b200_ctx* ctx, uint64_t bytes, void** ptr);
int b200_free(b200_ctx* ctx, void* ptr);
/* Pinned host staging (the reference maps host tensors with cudaHostRegister, buffer_cuda.cc:188). */
int b200_host_alloc(b200_ctx* ctx, uint64_t bytes, void** ptr);
int b200_host_free(b200_ctx* ctx, void* ptr);
/* Host-accessible (managed) allocation: what the reference's CUDA Buffer hands out for Buffer::Config::hostAccessible
 * (src/memory/buffer_cuda.cc:49-58), zero-filled. Freed with b200_free. */
int b200_malloc_managed(b200_ctx* ctx, uint64_t bytes, void** ptr);
/* Zero-copy mapping of an existing page-aligned host allocation onto the device (Tensor(device, cpuTensor),
 * src/memory/buffer_cuda.cc:140-200): pins it unless somebody already did; *registered tells the caller whether it owns
 * the registration (and must call b200_host_unregister). */
int b200_host_register(b200_ctx* ctx, void* host, uint64_t bytes, int* registered);
int b200_host_unregister(b200_ctx* ctx, void* host);
/* Tensor::copyFrom, src/memory/buffer_cuda.cc:284-306. kind: 0 h2d, 1 d2h, 2 d2d, 3 by address (UVA). Async on stream. */
int b200_memcpy(b200_ctx* ctx, void* dst, const void* src, uint64_t bytes, int kind, b200_stream stream);
int b200_memset(b200_ctx* ctx, void* dst, int value, uint64_t bytes, b200_stream stream);

/* src/runtime/native/cuda/impl.cc:35-118 (one non-blocking stream per runtime segment; sync at :244). */
int b200_stream_create(b200_ctx* ctx, b200_stream* stream);
int b200_stream_destroy(b200_ctx* ctx, b200_stream stream);
int b200_stream_synchronize(b200_ctx* ctx, b200_stream stream);
/* Per-module timing events of the runtime (src/runtime/native/cuda/impl.cc:96-118,206-262) and its post-submit check
 * of the thread's asynchronous CUDA error state (:228-231). */
int b200_event_create(b200_ctx* ctx, b200_event* event);
int b200_event_record(b200_ctx* ctx, b200_event event, b200_stream stream);
int b200_event_elapsed_ms(b200_ctx* ctx, b200_event start, b200_event end, float* ms);
int b200_event_destroy(b200_ctx* ctx, b200_event event);
int b200_check_async_error(b200_ctx* ctx);

/* ---- module compute(): one call per reference computeSubmit() --------------------------- */

/* window — src/domains/dsp/window/module_impl_native_cpu.cc:20-37.
 * Blackman taps evaluated in F64, stored as CF32 (imag 0); n == 1 -> 1+0i. out: [n] CF32. */
int b200_window_blackman_cf32(b200_ctx* ctx, b200_cf32* out, uint64_t n, b200_stream stream);

/* invert — src/domains/dsp/invert/module_impl_native_cpu.cc:78-103.
 * out = in * (-1)^k along an axis of even length `n` (k = axis coordinate), or the F64-evaluated
 * phasor exp(j*2*pi*floor(n/2)*k/n) for odd n. Tensor viewed as [outer, n, inner], contiguous. */
int b200_invert_cf32(b200_ctx* ctx, const b200_cf32* in, b200_cf32* out,
                     uint64_t outer, uint64_t n, uint64_t inner, b200_stream stream);

/* multiply — src/domains/core/multiply/module_impl_native_cpu.cc:86-100 with the NumPy broadcast
 * plan of module_impl.cc:28-83. Strides are in ELEMENTS of the broadcast views (0 on broadcast
 * dims), rank <= 8; c is contiguous row-major over `shape`. */
int b200_multiply_cf32(b200_ctx* ctx, const b200_cf32* a, const b200_cf32* b, b200_cf32* c,
                       int rank, const uint64_t* shape, const uint64_t* stride_a,
                       const uint64_t* stride_b, b200_stream stream);
int b200_multiply_f32(b200_ctx* ctx, const float* a, const float* b, float* c,
                      int rank, const uint64_t* shape, const uint64_t* stride_a,
                      const uint64_t* stride_b, b200_stream stream);

/* multiply_constant — src/domains/core/multiply_constant/module_impl_native_cpu.cc:82-100. */
int b200_multiply_constant_cf32(b200_ctx* ctx, const b200_cf32* in, b200_cf32* out, uint64_t count,
                                float constant, b200_stream stream);
int b200_multiply_constant_f32(b200_ctx* ctx, const float* in, float* out, uint64_t count,
                               float constant, b200_stream stream);

/* fft — src/domains/dsp/fft/module_impl_native_cpu.cc:129-140 (pocketfft::c2c, scale 1.0 in both
 * directions, forward sign exp(-j2*pi*kn/N)). Batched 1-D C2C over the last (contiguous) axis:
 * in/out [batch, n] CF32; in == out allowed. Any n >= 1: powers of two up to 8192 run the single-pass TMA-staged
 * register-radix kernel; 16384 / 32768 / 65536 a tiled two-pass plan (column tiles by 2-D TMA + 256-point rows with
 * 128-byte transposed runs over an L2-resident scratch), 131072 a radix-16 column pass + 8192-point rows, larger powers
 * of two a four-step plan (transposes + two batched sub-transforms); every
 * other length Bluestein's chirp-z through a power-of-two convolution (pocketfft does the same for large primes). Replaces cufftMakePlanMany64 + cufftExecC2C of
 * src/domains/dsp/fft/module_impl_native_cuda.cc:321-333,433. */
int b200_fft_plan_c2c(b200_ctx* ctx, uint64_t n, uint64_t batch, b200_fft_plan** plan);
int b200_fft_exec(b200_fft_plan* plan, const b200_cf32* in, b200_cf32* out, int forward,
                  b200_stream stream);
int b200_fft_plan_destroy(b200_fft_plan* plan);

/* Real-input transforms (pocketfft::r2c / r2r_fftpack, src/domains/dsp/fft/module_impl_native_cpu.cc:142-167) are
 * composed from the C2C kernels plus these layout steps over [batch, n] rows:
 *   op 0: full CF32 spectrum -> first n/2+1 bins (R2C output, `complexOutput`)
 *   op 1: full CF32 spectrum -> FFTPACK half-complex F32 [Re X0, Re X1, Im X1, ..., (Re X_{n/2})]
 *   op 2: FFTPACK half-complex F32 -> full Hermitian CF32 spectrum (input of the inverse)
 *   op 3: CF32 -> real part F32 */
int b200_fft_real_helper(b200_ctx* ctx, int op, const void* in, void* out, uint64_t batch, uint64_t n,
                         b200_stream stream);

/* Forward transform of REAL rows of even length 2h through one complex transform of length h (the row itself is the
 * even/odd-packed CF32 input) and one unpack kernel: 16 bytes of traffic per real sample instead of the 40 of
 * cast -> full C2C -> pack. `half_plan` = b200_fft_plan_c2c(ctx, h, batch); in [batch, 2h] F32 (8-byte aligned);
 * layout 0: out [batch, h + 1] CF32 (pocketfft::r2c, `complexOutput`), layout 1: out [batch, 2h] F32 FFTPACK
 * half-complex (pocketfft::r2r_fftpack) — src/domains/dsp/fft/module_impl_native_cpu.cc:142-167. For power-of-two
 * 32 <= h <= 8192 and a 16-byte aligned input the unpack runs in the transform kernel's own epilogue (one kernel, 8 bytes
 * of traffic per real sample); otherwise the plan owns a [batch, h] work buffer (allocated on first use). Odd lengths and
 * the inverse keep the composed path above. */
int b200_fft_exec_real(b200_fft_plan* half_plan, const float* in, void* out, int layout, b200_stream stream);

/* amplitude — src/domains/dsp/amplitude/module_impl_native_cpu.cc:73-99 with Backend::ApproxLog10
 * (include/jetstream/backend/devices/cpu/helpers.hh:61-74): out = |x|==0 ? -inf :
 * 20*ApproxLog10(|x|) + coeff, coeff = 20*log10f(1/N) (src/domains/dsp/amplitude/module_impl.cc:49-51).
 * Same operation order as the reference, no FMA contraction: bit-identical for finite input. */
int b200_amplitude_cf32(b200_ctx* ctx, const b200_cf32* in, float* out, uint64_t count, float coeff,
                        b200_stream stream);
int b200_amplitude_f32(b200_ctx* ctx, const float* in, float* out, uint64_t count, float coeff,
                       b200_stream stream);

/* Host-side coefficient helpers (pure functions, no device work):
 * amplitude scalingCoeff = 20 * log10f(1.0f / (float)n)      src/domains/dsp/amplitude/module_impl.cc:49-51
 * range scale/offset     = RangeImpl::updateCoefficients     src/domains/core/range/module_impl.cc:51-63 */
int b200_amplitude_scaling_coeff(uint64_t n, float* coeff);
int b200_range_coefficients(float min, float max, float* scale, float* offset);

/* range ("Scale") — src/domains/core/range/module_impl_native_cpu.cc:67-82:
 * out = scale == 0 ? 0.5 : 0.5 + 0.5*tanhf(4*((in*scale + offset) - 0.5)); scale/offset from
 * RangeImpl::updateCoefficients (src/domains/core/range/module_impl.cc:51-63). */
int b200_range_f32(b200_ctx* ctx, const float* in, float* out, uint64_t count, float scale,
                   float offset, b200_stream stream);

/* Layout gather / scatter: strided element copy over `shape` (rank <= 8, strides in ELEMENTS, elem_bytes 1, 2, 4 or 8).
 * The role of the reference's `fft_layout` kernel, src/domains/dsp/fft/module_impl_native_cuda.cc:31-141: modules that
 * declare Module::Taint::DISCONTIGUOUS bring strided / non-innermost-axis views into the contiguous [batch, n]
 * layout of the fast kernels with it and scatter the result back. */
int b200_copy_strided(b200_ctx* ctx, const void* src, void* dst, int elem_bytes, int rank, const uint64_t* shape,
                      const uint64_t* src_stride, const uint64_t* dst_stride, b200_stream stream);

/* cast F32 -> CF32 (imag 0) — src/domains/core/cast/module_impl_native_cpu.cc (CF32 input bypasses). */
int b200_cast_f32_cf32(b200_ctx* ctx, const float* in, b200_cf32* out, uint64_t count, b200_stream stream);

/* agc — tiled RMS automatic gain control, src/domains/dsp/agc/module_impl_native_cpu.cc:76-160 (AgcImpl config:
 * include/jetstream/domains/dsp/agc/module.hh:8-19; validation module_impl.cc:7-45). in/out are [lanes, samples]
 * contiguous (sample axis innermost), F32 (is_complex = 0) or CF32. All gain arithmetic in F64 as the reference.
 * `scratch` is caller-owned device memory of b200_agc_scratch_bytes() bytes. Stateless across calls. */
int b200_agc_scratch_bytes(uint64_t lanes, uint64_t samples, uint64_t tile_size, uint64_t* bytes);
int b200_agc(b200_ctx* ctx, const void* in, void* out, int is_complex, uint64_t lanes, uint64_t samples,
             uint64_t tile_size, double reference, double epsilon, double min_gain, double max_gain,
             double max_gain_change, void* scratch, b200_stream stream);

/* cast integer -> F32 / complex integer -> CF32 — src/domains/core/cast/module_impl_native_cpu.cc:163-330 with the
 * scaler of module_impl.cc:50-72: out = (F32)in / 128 (I8, U8, CI8, CU8), / 32768 (16-bit), / 2147483648 (32-bit).
 * Unsigned types are NOT re-centred (the reference does not either). `count` is in ELEMENTS of `in_dtype`
 * (a complex element is two scalars); `out` holds count F32 or count CF32. */
#define B200_DTYPE_F32   0
#define B200_DTYPE_CF32  1
#define B200_DTYPE_I8    2
#define B200_DTYPE_U8    3
#define B200_DTYPE_I16   4
#define B200_DTYPE_U16   5
#define B200_DTYPE_I32   6
#define B200_DTYPE_U32   7
#define B200_DTYPE_CI8   8
#define B200_DTYPE_CU8   9
#define B200_DTYPE_CI16  10
#define B200_DTYPE_CU16  11
#define B200_DTYPE_CI32  12
#define B200_DTYPE_CU32  13
int b200_cast_int(b200_ctx* ctx, const void* in, int in_dtype, void* out, uint64_t count, b200_stream stream);

/* ---- fused spectral chain: the spectrum_engine block ------------------------------------ */

/* Replaces the module sequence wired by SpectrumEngineImpl::create
 * (src/domains/dsp/spectrum_engine/block_impl.cc:120-217): multiply(x, window) -> fft(forward) ->
 * amplitude -> [range], in ONE kernel: x is read once (8 B/sample), the F32 result written once
 * (4 B/sample). `window` is the [n] CF32 tensor the block's window->invert->reshape modules
 * produce (already sign-flipped); it is captured at plan creation (static, settled output).
 *   x   : [batch, n] CF32 contiguous, 16-byte aligned       out : [batch, n] F32
 *   amp_coeff = 20*log10f(1/n); enable_range != 0 applies range(scale, offset).
 * Powers of two 2 <= n <= 8192 run ONE fused kernel (n == 4096: fft4096_kernel; 16..8192: fft_radix_kernel;
 * 2..8: fft_generic_kernel); n = 16384 / 32768 / 65536 run TWO fused kernels over the tiled two-pass plan (window in the
 * column pass, amplitude / range in the row pass; any batch <= or > max_batch, processed in 64 MB chunks). Any other
 * length runs the module sequence multiply -> fft -> amplitude -> range through a plan-owned scratch (exec must then
 * use batch == max_batch).
 * Amplitude domain of the dB output (the epilogue forms |X|^2 in F32 before an approximate square root, and adds no
 * branch for either limit):
 *   |X| > sqrt(F32 max) ~ 1.8e19 (a coherent CF32 tone of about 1e16 per sample): |X|^2 overflows to +inf and the bin
 *     reads 20 ApproxLog10(2^128) + amp_coeff ~ 770.6 dB + amp_coeff, where the reference gives 20 log10|X| + amp_coeff,
 *     300 to 400 dB lower;
 *   2^-75 < |X| < 2^-63 ~ 1.1e-19: |X|^2 is subnormal, the square root flushes it to zero and the bin reads
 *     20 ApproxLog10(2^-127) + amp_coeff ~ -764.6 dB + amp_coeff; below about 2^-75 |X|^2 is 0 and the bin reads -inf.
 * The range output saturates to 1.0 above and to 0.0 below either way. Integer inputs cannot reach the upper limit.
 * A NaN sample makes its row's spectrum NaN, and every bin of that row then reads 20 ApproxLog10((1 - 2^-24) 2^129) +
 * amp_coeff ~ 776.7 dB + amp_coeff (range: 1.0) where the reference gives NaN. */
int b200_chain_plan_create(b200_ctx* ctx, uint64_t n, uint64_t max_batch, const b200_cf32* window_dev,
                           b200_chain_plan** plan);
int b200_chain_exec(b200_chain_plan* plan, const b200_cf32* x, float* out, uint64_t batch,
                    float amp_coeff, int enable_range, float scale, float offset, b200_stream stream);
/* The same chain reading complex-integer samples (in_dtype = B200_DTYPE_CI8 ... CU32; B200_DTYPE_CF32 forwards to
 * b200_chain_exec): the `cast` module that precedes spectrum_engine in an SDR flowgraph
 * (src/domains/core/cast/module_impl_native_cpu.cc:270-330) folded into the kernel's load. n = 4096 with a real
 * window and CI8/CU8/CI16/CU16 input is ONE kernel (2 or 4 B/sample read instead of cast's 2+8 write/read);
 * everything else runs b200_cast_int into a plan-owned scratch and then the CF32 chain. Results are bit-identical
 * to cast -> b200_chain_exec. */
int b200_chain_exec_typed(b200_chain_plan* plan, const void* x, int in_dtype, float* out, uint64_t batch,
                          float amp_coeff, int enable_range, float scale, float offset, b200_stream stream);

/* spectrum_engine with enableAgc (src/domains/dsp/spectrum_engine/block_impl.cc:186-200: an `agc` module with one
 * RMS tile per spectrum between fft and amplitude), still ONE kernel: the row's mean power comes from the windowed
 * input by Parseval, gain = clamp(reference / sqrt(mean |X|^2 + epsilon), min_gain, max_gain) in F64 as
 * AgcImplNativeCpu (module_impl_native_cpu.cc:112-124; the rate limit does not apply to a single tile).
 * n = 4096 with a real window only (ERROR otherwise: wire fft -> agc -> amplitude -> range instead);
 * in_dtype CF32 or CI8/CU8/CI16/CU16. */
int b200_chain_exec_agc(b200_chain_plan* plan, const void* x, int in_dtype, float* out, uint64_t batch, float amp_coeff,
                        int enable_range, float scale, float offset, double agc_reference, double agc_epsilon,
                        double agc_min_gain, double agc_max_gain, b200_stream stream);

/* spectrum_engine -> lineplot without a second pass over the spectra: the chain output AND colsum[n] = sum over the batch
 * of every output column (the first loop of LineplotImplNativeCpu::computeSubmit,
 * src/domains/visualization/lineplot/module_impl_native_cpu.cc:93-98). n = 4096 with a real window and CF32 / CI8 / CU8 /
 * CI16 / CU16 input: the running sums are kept in the kernel's registers (two extra FADD per output pair); every other
 * plan runs the chain and then the row-split column-sum kernel. Feed colsum to b200_lineplot_update_from_colsum.
 * The sums are F32 in a fixed order, so they are reproducible run to run (a reassociation of the reference's
 * sequential sum over the batch):
 *   fused form: CTA b of G = min(batch, 2 SMs) adds out rows b, b + G, b + 2G, ... in that order, starting from +0;
 *     then colsum[e] = partial[0][e] + partial[1][e] + ... + partial[G-1][e], in that order, starting from +0;
 *   row-split form (dense aligned rows): splits = max(1, min(ceil(4 SMs / column_blocks), ceil(batch / 64))) with
 *     column_blocks = ceil(n / 1024); split s adds rows s R ... min(batch, (s + 1) R) - 1 in order from +0, with
 *     R = ceil(batch / splits); colsum[e] adds the splits in order 0 ... splits - 1 from +0.
 * batch == 0 sets colsum to +0. */
int b200_chain_exec_colsum(b200_chain_plan* plan, const void* x, int in_dtype, float* out, uint64_t batch, float amp_coeff,
                           int enable_range, float scale, float offset, float* colsum, b200_stream stream);

/* Same computation for HOST-resident tensors (what the reference's TestContext hands a CUDA module:
 * host memory mapped onto the device, src/testing.cc:136, src/memory/buffer_cuda.cc:188). x_host and
 * out_host should be pinned (b200_host_alloc) for full PCIe rate. The batch is cut into chunks of
 * `chunk_rows` rows (0 = 128 MiB of input) and pipelined H2D -> kernel -> D2H on three streams with three
 * device staging slots. SYNCHRONOUS: returns when out_host is complete. */
int b200_chain_exec_host(b200_chain_plan* plan, const b200_cf32* x_host, float* out_host, uint64_t batch,
                         float amp_coeff, int enable_range, float scale, float offset, uint64_t chunk_rows);
/* The same pipeline for complex-integer host samples (in_dtype = B200_DTYPE_CI8 ... CU32; CF32 forwards): an SDR's
 * native 8 / 16-bit samples cross PCIe at 2 / 4 bytes instead of 8 and are converted inside the kernel's load
 * (b200_chain_exec_typed). Results are bit-identical to cast -> b200_chain_exec_host. */
int b200_chain_exec_host_typed(b200_chain_plan* plan, const void* x_host, int in_dtype, float* out_host, uint64_t batch,
                               float amp_coeff, int enable_range, float scale, float offset, uint64_t chunk_rows);
int b200_chain_plan_destroy(b200_chain_plan* plan);
/* Name of the kernel variant exec() launches for this plan (for logs / profiles). */
const char* b200_chain_plan_variant(const b200_chain_plan* plan);

/* ---- lineplot / waterfall consumers (SURVEY.md 8 f1) ------------------------------------------------------------- */

/* lineplot — LineplotImplNativeCpu::computeSubmit, src/domains/visualization/lineplot/module_impl_native_cpu.cc:80-122
 * (geometry of LineplotImpl::validate, module_impl.cc:95-187; CUDA counterpart module_impl_native_cuda.cc:21-60):
 *   sum[e]  = sum_b in[b * batch_stride + e * decimation * element_stride]        e < elements = extent / decimation
 *   amp     = fmin(fmax(sum[e] * normalization - 1, -1), 1)                        normalization = 1 / (0.5 * batches)
 *   average[e] -= average[e] / averaging;  average[e] += amp / averaging;  points[2 e + 1] = average[e]
 * `average` [elements] is the module's persistent state, `points` [elements, 2] the signalPoints tensor (x in column 0,
 * written once by b200_lineplot_init: e * 2.0f / (elements - 1) - 1.0f). Strides in ELEMENTS. The batch sum is a
 * row-split partial sum + fixed-order reduction (reassociated vs the reference's sequential loop; identical for
 * batches <= 64). `scratch`: b200_lineplot_scratch_bytes() bytes of device memory. */
int b200_lineplot_scratch_bytes(uint64_t batches, uint64_t elements, uint64_t decimation, uint64_t* bytes);
int b200_lineplot_init(b200_ctx* ctx, float* points, float* average, uint64_t elements, b200_stream stream);
int b200_lineplot_update(b200_ctx* ctx, const float* in, uint64_t batches, uint64_t elements, uint64_t batch_stride,
                         uint64_t element_stride, uint64_t decimation, float normalization, uint64_t averaging,
                         float* average, float* points, void* scratch, b200_stream stream);
/* The same update from column sums that already exist (b200_chain_exec_colsum): colsum is indexed e * decimation. */
int b200_lineplot_update_from_colsum(b200_ctx* ctx, const float* colsum, uint64_t elements, uint64_t decimation,
                                     float normalization, uint64_t averaging, float* average, float* points,
                                     b200_stream stream);

/* waterfall — WaterfallImplNativeCpu::computeSubmit, src/domains/visualization/waterfall/module_impl_native_cpu.cc:53-78
 * with PlanWaterfallWrite / WaterfallRingState::advance (waterfall/ring_state.hh:18-44): the newest min(batches, height)
 * input rows go to ring rows (write_index + ...) % height; ring is [height, elements] F32. Bit-exact (a copy).
 * b200_waterfall_advance is the host-side cursor update the caller applies after each update. */
int b200_waterfall_update(b200_ctx* ctx, const float* in, uint64_t batches, uint64_t elements, uint64_t batch_stride,
                          uint64_t element_stride, float* ring, uint64_t height, uint64_t write_index,
                          b200_stream stream);
int b200_waterfall_advance(uint64_t* write_index, uint64_t batches, uint64_t height);

/* ---- filter block ---------------------------------------------------------------------------- */

/* filter_taps — FilterTapsImplNativeCpu::generateCoeffs, src/domains/dsp/filter_taps/module_impl_native_cpu.cc:46-80
 * (validation of src/domains/dsp/filter_taps/module_impl.cc:12-105). STATIC_OUTPUT, evaluated once, on the
 * host, in F64 with the reference's own formula; out_host: [heads, taps] CF32. */
int b200_filter_taps_host(double sample_rate, double bandwidth, const double* center, uint64_t heads,
                          uint64_t taps, b200_cf32* out_host);

/* Streaming (decimating) FIR = the per-cycle module chain of the `filter` block
 * (src/domains/dsp/filter/block_impl.cc:350-582: pad -> fft -> multiply -> fold -> ifft -> multiply_constant ->
 * unpad -> overlap_add) evaluated in the time domain: y[q] = sum_k h[k] xs[q R - k] over the time-continuous
 * stream of frames; `decimation` = R (1 when the block does not resample, block_impl.cc:64-90).
 *   taps_host : [heads, ntaps] CF32 on the HOST (captured by the plan)
 *   x         : [frames, frame_len] CF32 device, frames consecutive in time
 *   y         : [frames, heads, frame_len / R] CF32 device
 * The plan carries the last ntaps-1 input samples across calls (the reference carries the (ntaps-1)/R
 * output tail in overlap_add, module_impl_native_cpu.cc:155-198); b200_fir_reset zeroes it. */
int b200_fir_plan_create(b200_ctx* ctx, const b200_cf32* taps_host, uint64_t ntaps, uint64_t heads,
                         uint64_t decimation, b200_fir_plan** plan);
/* The kernel forms exec() can launch for this plan (for logs / tests): the 8-byte sample form, and the 16-byte chunk-pair
 * form when the plan has one, e.g. "sample OB=7 threads=64 taps=const real qt=448 ctas=792; pair OB=5 threads=128
 * taps=const real qt=640 ctas=528". OB = outputs per thread, qt = outputs per tile, taps = tap table in the kernel
 * parameters or in shared memory, ctas = most CTAs one launch uses. A call takes the pair form only when its input is
 * 16-byte aligned and of even length, so the string says what is eligible, not what a given call ran. */
const char* b200_fir_plan_variant(const b200_fir_plan* plan);
/* Frequency-translating heads = the block's fold offsets + phase_correction module (block_impl.cc:118-160,
 * 519-532; src/domains/dsp/fold/module_impl_native_cpu.cc:130-147; src/domains/dsp/phase_correction/
 * module_impl_native_cpu.cc:81-115): head h is shifted down by center_bins[h] bins of the block's M-point spectrum
 * (M = frame_len + ntaps - 1) before decimation; the per-frame phase is carried across calls in F64. */
int b200_fir_plan_set_translation(b200_fir_plan* plan, uint64_t frame_len, const int64_t* center_bins);
int b200_fir_exec(b200_fir_plan* plan, const b200_cf32* x, b200_cf32* y, uint64_t frames, uint64_t frame_len,
                  b200_stream stream);
int b200_fir_reset(b200_fir_plan* plan, b200_stream stream);
/* Time sharding (one stream cut into slabs for several GPUs, SURVEY.md §8e): load the halo — the last `count` <= taps-1
 * input samples that precede this plan's slab (device pointer) — as the carried state that overlap_add's tail is in the
 * reference (src/domains/dsp/overlap_add/module_impl_native_cpu.cc:155-198). `frames_before` = frames of the stream
 * before the slab (only used by translating plans: phase_correction continues from there). */
int b200_fir_set_history(b200_fir_plan* plan, const b200_cf32* tail_dev, uint64_t count, uint64_t frames_before,
                         b200_stream stream);
int b200_fir_plan_destroy(b200_fir_plan* plan);

/* The separate stages of the filter / filter_engine wiring (src/domains/dsp/filter/block_impl.cc:350-582), for the
 * layouts the fused FIR does not take and for flowgraphs wired by hand. pad and unpad are b200_copy_strided calls. */

/* fold — FoldImplNativeCpu::foldKernel, src/domains/dsp/fold/module_impl_native_cpu.cc:102-172 (validation and offsets:
 * src/domains/dsp/fold/module_impl.cc:8-113). in: contiguous [outer, axis, inner], out: contiguous [outer, size, inner],
 * F32 (is_complex = 0) or CF32; `size` divides `axis`, R = axis / size:
 *   out[r, o, i] = (1/R) sum_{g < R} in[r, (o + g size - offset) mod axis, i]
 * summed in F64 in ascending g, divided by R in F64 and rounded once: bit-identical to the reference. `offset` is the
 * module's scalar offset; with `channel_offsets` (device pointer, `channels` U64 values, the input's "channelOffsets"
 * attribute) output element k uses channel_offsets[(k / channel_inner) % channels] instead. Offsets are taken mod axis.
 * Stateless. */
int b200_fold(b200_ctx* ctx, const void* in, void* out, int is_complex, uint64_t outer, uint64_t axis, uint64_t inner,
              uint64_t size, uint64_t offset, const uint64_t* channel_offsets, uint64_t channels,
              uint64_t channel_inner, b200_stream stream);

/* overlap_add — OverlapAddImplNativeCpu, src/domains/dsp/overlap_add/module_impl_native_cpu.cc:120-202. buffer / out:
 * contiguous [outer, buffer_len, inner]; overlap: contiguous [outer, overlap_len, inner], overlap_len <= buffer_len;
 * F32 (is_complex = 0) or CF32. The batch coordinate of overlap element k is (k / batch_stride) % batches (batches = 1
 * without a batch axis). out = buffer, and over the first overlap_len samples of every row out += the previous batch's
 * overlap, or for batch 0 the carried `previous` tail ([overlap with the batch extent reduced to 1], device memory
 * owned by the caller, zero before the first call). Then `previous` = the last batch of overlap. One F32 add per
 * element: bit-identical to the reference. Two launches on `stream`, so the read of the old tail is ordered before its
 * overwrite; `previous` must not alias the other tensors. */
int b200_overlap_add(b200_ctx* ctx, const void* buffer, const void* overlap, void* out, void* previous, int is_complex,
                     uint64_t outer, uint64_t buffer_len, uint64_t overlap_len, uint64_t inner, uint64_t batches,
                     uint64_t batch_stride, b200_stream stream);

/* phase_correction — PhaseCorrectionImplNativeCpu::computeSubmit, src/domains/dsp/phase_correction/
 * module_impl_native_cpu.cc:81-115. in / out: contiguous CF32, `count` elements; element k belongs to batch
 * (k / batch_inner) % batches and channel (k / channel_inner) % channels (batches = 1 / channels = 1 without the axis)
 * and is multiplied, with std::complex<float>'s operation order, by (cos phi, sin phi) rounded to F32 from
 *   phi = phases[channel] + wrapped_increments[channel] * batch      (F64, no FMA)
 * `phases` and `wrapped_increments` are HOST arrays of `channels` values, passed to the kernel by value: the caller
 * keeps the per-channel phase on the host and advances it after each call as the reference does
 * (phases[c] = remainder(phases[c] + wrapped[c] * batches, 2 pi)). Differs from the reference only where CUDA's F64
 * cos / sin and glibc's round to different F32 values. At most B200_PHASE_CORRECTION_MAX_CHANNELS channels. */
#define B200_PHASE_CORRECTION_MAX_CHANNELS 128
int b200_phase_correction(b200_ctx* ctx, const b200_cf32* in, b200_cf32* out, uint64_t count, uint64_t batches,
                          uint64_t batch_inner, uint64_t channels, uint64_t channel_inner, const double* phases,
                          const double* wrapped_increments, b200_stream stream);

/* ---- fm ---------------------------------------------------------------------------------------- */

/* fm — FmImplNativeCpu::computeSubmit, src/domains/dsp/fm/module_impl_native_cpu.cc:43-175, coefficients of
 * src/domains/dsp/fm/module_impl.cc:108-155. x: [frames, lanes, frame_len] CF32 (frames consecutive in time,
 * lanes independent). out: same shape F32 (narrow) or [frames, lanes, frame_len, 2] = left/right (wide != 0:
 * pilot NCO + pilot recovery, notch + 3 low-pass biquads on the sum and difference paths, evaluated as blocked
 * linear-recurrence scans). deemphasis_us: 0 (none), 50 or 75. Per-lane state lives in the plan. */
int b200_fm_plan_create(b200_ctx* ctx, uint64_t lanes, float sample_rate, int wide, int deemphasis_us,
                        b200_fm_plan** plan);
int b200_fm_exec(b200_fm_plan* plan, const b200_cf32* x, float* out, uint64_t frames, uint64_t frame_len,
                 b200_stream stream);
int b200_fm_reset(b200_fm_plan* plan, b200_stream stream);
int b200_fm_plan_destroy(b200_fm_plan* plan);
/* Host-only: the wideband decoder's pilot NCO phases (F32 running sum with wrap, fm/module_impl_native_cpu.cc:172-175) of
 * samples n0 .. n0 + len - 1 since reset, reconstructed from the orbit table the plan uses on the device instead of a
 * serial walk (the F32 state is periodic: *pre transient samples, then *cycle samples repeating). out may be NULL. */
int b200_fm_nco_phases_host(float sample_rate, uint64_t n0, uint64_t len, float* out, uint64_t* pre, uint64_t* cycle);
/* Test / diagnostic hook: the same phases generated on the device by the kernel b200_fm_exec uses, for a wideband
 * plan: out is a device buffer of len F32 (a wrong fold moves a phase by a few ulps, below what the demodulated output
 * can show, so tests compare these bit for bit with b200_fm_nco_phases_host). b200_fm_exec takes the phases of its samples from n0 = the number of samples per lane it has
 * demodulated since the plan's creation or last reset. */
int b200_fm_nco_phases(b200_fm_plan* plan, uint64_t n0, uint64_t len, float* out, b200_stream stream);

#ifdef __cplusplus
}
#endif

#endif /* B200DSP_H */
