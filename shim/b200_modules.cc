// Reference-side binding for the "b200" provider: Module::Impl subclasses that derive the reference's own
// shared module implementations (validate/define/create/reconfigure are the reference's code, unchanged) and
// forward computeSubmit(stream) to libb200dsp through the C ABI (include/b200dsp.h).
//
// This is the file a CyberEther maintainer would add (e.g. as src/domains/b200/modules.cc, or as a `.cep`
// plugin target with `device: cuda`, docs/plugins.md:89-112). It is compiled here against the reference
// headers where they lie (oracle/build_shim.sh) to prove the boundary; it contains no kernels.
//
//   registration     JST_REGISTER_MODULE(Impl, DeviceType::CUDA, RuntimeType::NATIVE, "b200")
//                                                                     include/jetstream/registry.hh:174-175
//   compute hooks    NativeCudaRuntimeContext::{computeInitialize, computeSubmit(const cudaStream_t&),
//                    computeDeinitialize}                              include/jetstream/runtime_context_native_cuda.hh:13-39
//   selection        blockCreate(name, type, config, inputs, DeviceType::CUDA, RuntimeType::NATIVE, "b200")
//                    or `device: cuda / runtime: native / provider: b200` in a flowgraph YAML
#include <cmath>
#include <any>
#include <cstdint>
#include <memory>
#include <vector>

#include <jetstream/backend/base.hh>
#include <jetstream/logger.hh>
#include <jetstream/module_context.hh>
#include <jetstream/registry.hh>
#include <jetstream/runtime_context_native_cuda.hh>
#include <jetstream/scheduler_context.hh>

#include "domains/core/cast/module_impl.hh"
#include "domains/core/expand_dims/module_impl.hh"
#include "domains/core/multiply/module_impl.hh"
#include "domains/core/multiply_constant/module_impl.hh"
#include "domains/core/pad/module_impl.hh"
#include "domains/core/range/module_impl.hh"
#include "domains/core/reshape/module_impl.hh"
#include "domains/core/unpad/module_impl.hh"
#include "domains/dsp/agc/module_impl.hh"
#include "domains/dsp/amplitude/module_impl.hh"
#include "domains/dsp/fft/module_impl.hh"
#include "domains/dsp/filter_taps/module_impl.hh"
#include "domains/dsp/fm/module_impl.hh"
#include "domains/dsp/fold/module_impl.hh"
#include "domains/dsp/invert/module_impl.hh"
#include "domains/dsp/overlap_add/module_impl.hh"
#include "domains/dsp/phase_correction/module_impl.hh"
#include "domains/dsp/window/module_impl.hh"
#include "domains/visualization/lineplot/module_impl.hh"
#include "domains/visualization/waterfall/module_impl.hh"

#include "b200_provider.hh"

namespace Jetstream::Modules {

using B200::Check;
using B200::DevicePtr;
static inline b200_ctx* B200Ctx() { return B200::Ctx(); }

// ---- window ---------------------------------------------------------------------------------------
struct WindowImplB200 : public WindowImpl, public NativeCudaRuntimeContext, public Scheduler::Context {
    Result computeSubmit(const cudaStream_t& stream) override {
        return Check(b200_window_blackman_cf32(B200Ctx(), DevicePtr<b200_cf32>(output), size, stream), "WINDOW");
    }
};
JST_REGISTER_MODULE(WindowImplB200, DeviceType::CUDA, RuntimeType::NATIVE, "b200");

// ---- invert ---------------------------------------------------------------------------------------
struct InvertImplB200 : public InvertImpl, public NativeCudaRuntimeContext, public Scheduler::Context {
    Result create() final {
        JST_CHECK(InvertImpl::create());
        if (!input.contiguous() || input.dtype() != DataType::CF32) {
            JST_ERROR("[MODULE_INVERT_B200] Only contiguous CF32 inputs are supported by this provider.");
            return Result::ERROR;
        }
        outer = 1;
        inner = 1;
        for (Index i = 0; i < resolvedAxis; ++i) outer *= input.shape(i);
        for (Index i = resolvedAxis + 1; i < input.rank(); ++i) inner *= input.shape(i);
        return Result::SUCCESS;
    }
    Result computeSubmit(const cudaStream_t& stream) override {
        return Check(b200_invert_cf32(B200Ctx(), DevicePtr<b200_cf32>(input), DevicePtr<b200_cf32>(output), outer,
                                      input.shape(resolvedAxis), inner, stream), "INVERT");
    }
    U64 outer = 1, inner = 1;
};
JST_REGISTER_MODULE(InvertImplB200, DeviceType::CUDA, RuntimeType::NATIVE, "b200");

// ---- reshape / cast (views; cast bypasses when the dtype already matches) ----------------------------
struct ReshapeImplB200 : public ReshapeImpl, public NativeCudaRuntimeContext, public Scheduler::Context {
    Result computeSubmit(const cudaStream_t&) override { return Result::SUCCESS; }
};
JST_REGISTER_MODULE(ReshapeImplB200, DeviceType::CUDA, RuntimeType::NATIVE, "b200");

struct CastImplB200 : public CastImpl, public NativeCudaRuntimeContext, public Scheduler::Context {
    Result computeSubmit(const cudaStream_t& stream) override {
        if (bypass) {
            return Result::SUCCESS;
        }
        if (input.dtype() == DataType::F32 && outputDtype == DataType::CF32 && input.contiguous()) {
            return Check(b200_cast_f32_cf32(B200Ctx(), DevicePtr<float>(input), DevicePtr<b200_cf32>(output),
                                            input.size(), stream), "CAST");
        }
        // integer -> F32 and complex integer -> CF32 (module_impl_native_cpu.cc:163-330); dtype codes of b200dsp.h
        const int code = B200::IntegerDtypeCode(input.dtype());
        const bool complexIn = code >= B200_DTYPE_CI8;
        if (code < 0 || !input.contiguous() || outputDtype != (complexIn ? DataType::CF32 : DataType::F32)) {
            JST_ERROR("[MODULE_CAST_B200] Unsupported conversion '{}' -> '{}' (contiguous inputs only).",
                      input.dtype(), outputDtype);
            return Result::ERROR;
        }
        return Check(b200_cast_int(B200Ctx(), DevicePtr<void>(input), code, DevicePtr<void>(output), input.size(),
                                   stream), "CAST");
    }
};
JST_REGISTER_MODULE(CastImplB200, DeviceType::CUDA, RuntimeType::NATIVE, "b200");

// ---- multiply ---------------------------------------------------------------------------------------
struct MultiplyImplB200 : public MultiplyImpl, public NativeCudaRuntimeContext, public Scheduler::Context {
    Result create() final {
        JST_CHECK(MultiplyImpl::create());
        const Index rank = c.rank();
        if (rank > 8) {
            JST_ERROR("[MODULE_MULTIPLY_B200] Rank {} exceeds the supported 8.", rank);
            return Result::ERROR;
        }
        shape.assign(c.shape().begin(), c.shape().end());
        strideA.assign(a.stride().begin(), a.stride().end());   // broadcast views: stride 0 on broadcast dims
        strideB.assign(b.stride().begin(), b.stride().end());
        return Result::SUCCESS;
    }
    Result computeSubmit(const cudaStream_t& stream) override {
        const int rank = static_cast<int>(shape.size());
        if (a.dtype() == DataType::CF32) {
            return Check(b200_multiply_cf32(B200Ctx(), DevicePtr<b200_cf32>(a), DevicePtr<b200_cf32>(b),
                                            DevicePtr<b200_cf32>(c), rank, shape.data(), strideA.data(),
                                            strideB.data(), stream), "MULTIPLY");
        }
        return Check(b200_multiply_f32(B200Ctx(), DevicePtr<float>(a), DevicePtr<float>(b), DevicePtr<float>(c), rank,
                                       shape.data(), strideA.data(), strideB.data(), stream), "MULTIPLY");
    }
    std::vector<U64> shape, strideA, strideB;
};
JST_REGISTER_MODULE(MultiplyImplB200, DeviceType::CUDA, RuntimeType::NATIVE, "b200");

// ---- fft ----------------------------------------------------------------------------------------------
// CF32 -> CF32 (either direction) through b200_fft_exec; F32 input, forward (pocketfft::r2c with `complexOutput`, else
// r2r_fftpack: src/domains/dsp/fft/module_impl_native_cpu.cc:142-167) through b200_fft_exec_real — one complex transform of
// half the length on the real row itself plus the unpack kernel.
// A CF32 transform along another axis, or over a strided view (the module is DISCONTIGUOUS), gathers the rows into a
// contiguous [rows, n] scratch with b200_copy_strided, transforms it in place and scatters it into the output — what the
// reference's CUDA module does with its fft_layout kernel (module_impl_native_cuda.cc:31-141).
struct FftImplB200 : public FftImpl, public NativeCudaRuntimeContext, public Scheduler::Context {
    Result create() final {
        JST_CHECK(FftImpl::create());
        const U64 n = input.shape(resolvedAxis);
        realInput = input.dtype() == DataType::F32;
        if (input.dtype() != DataType::CF32 && !realInput) {
            JST_ERROR("[MODULE_FFT_B200] Unsupported input data type.");
            return Result::ERROR;
        }
        const bool innermost = input.contiguous() && resolvedAxis + 1 == input.rank();
        if (realInput && !innermost) {
            JST_ERROR("[MODULE_FFT_B200] Real input: this provider implements contiguous transforms along the innermost axis.");
            return Result::ERROR;
        }
        if (realInput && (!forward || n < 4 || n % 2 != 0)) {
            JST_ERROR("[MODULE_FFT_B200] Real input: this provider implements the forward transform of even lengths >= 4.");
            return Result::ERROR;
        }
        gatherShape.clear();
        inputStride.clear();
        outputStride.clear();
        rows = Tensor();
        if (!innermost) {
            if (input.rank() > 8) {
                JST_ERROR("[MODULE_FFT_B200] Rank {} exceeds the supported 8.", input.rank());
                return Result::ERROR;
            }
            // input / output dimensions in the order (every other axis, transform axis); scratch strides row-major
            const auto& inStride = input.stride();
            const auto& outStride = output.stride();
            for (Index d = 0; d <= input.rank(); ++d) {
                const Index dim = d == input.rank() ? resolvedAxis : d;
                if (d == resolvedAxis) {
                    continue;
                }
                gatherShape.push_back(input.shape(dim));
                inputStride.push_back(inStride[dim]);
                outputStride.push_back(outStride[dim]);
            }
            rowStride.assign(gatherShape.size(), 1);
            for (size_t d = gatherShape.size() - 1; d > 0; --d) {
                rowStride[d - 1] = rowStride[d] * gatherShape[d];
            }
            JST_CHECK(rows.create(input.device(), DataType::CF32, {input.size() / n, n}));
        }
        return Result::SUCCESS;
    }
    Result computeInitialize() override {
        const U64 n = input.shape(resolvedAxis);
        return Check(b200_fft_plan_c2c(B200Ctx(), realInput ? n / 2 : n, input.size() / n, &plan), "FFT");
    }
    Result computeSubmit(const cudaStream_t& stream) override {
        if (realInput) {
            return Check(b200_fft_exec_real(plan, DevicePtr<float>(input), DevicePtr<void>(output), complexOutput ? 0 : 1, stream),
                         "FFT");
        }
        if (!gatherShape.empty()) {
            const int rank = static_cast<int>(gatherShape.size());
            auto* scratch = DevicePtr<b200_cf32>(rows);
            JST_CHECK(Check(b200_copy_strided(B200Ctx(), DevicePtr<b200_cf32>(input), scratch, 8, rank, gatherShape.data(),
                                              inputStride.data(), rowStride.data(), stream), "FFT"));
            JST_CHECK(Check(b200_fft_exec(plan, scratch, scratch, forward ? 1 : 0, stream), "FFT"));
            return Check(b200_copy_strided(B200Ctx(), scratch, DevicePtr<b200_cf32>(output), 8, rank, gatherShape.data(),
                                           rowStride.data(), outputStride.data(), stream), "FFT");
        }
        return Check(b200_fft_exec(plan, DevicePtr<b200_cf32>(input), DevicePtr<b200_cf32>(output), forward ? 1 : 0,
                                   stream), "FFT");
    }
    Result computeDeinitialize() override {
        const auto result = Check(b200_fft_plan_destroy(plan), "FFT");
        plan = nullptr;
        return result;
    }
    b200_fft_plan* plan = nullptr;
    bool realInput = false;
    Tensor rows;                                                   // [rows, n] gather scratch (other axes only)
    std::vector<U64> gatherShape, inputStride, outputStride, rowStride;
};
JST_REGISTER_MODULE(FftImplB200, DeviceType::CUDA, RuntimeType::NATIVE, "b200");

// ---- agc ---------------------------------------------------------------------------------------------------
struct AgcImplB200 : public AgcImpl, public NativeCudaRuntimeContext, public Scheduler::Context {
    Result create() final {
        JST_CHECK(AgcImpl::create());
        if (!input.contiguous() || sampleAxis + 1 != input.rank() ||
            (input.dtype() != DataType::CF32 && input.dtype() != DataType::F32)) {
            JST_ERROR("[MODULE_AGC_B200] This provider implements contiguous F32 / CF32 inputs with the sample axis innermost.");
            return Result::ERROR;
        }
        return Result::SUCCESS;
    }
    Result computeSubmit(const cudaStream_t& stream) override {
        const U64 samples = input.shape(sampleAxis);
        uint64_t need = 0;
        JST_CHECK(Check(b200_agc_scratch_bytes(laneCount, samples, tileSize, &need), "AGC"));
        if (need > scratchBytes) {                       // tileSize may be reconfigured between cycles
            b200_free(B200Ctx(), scratch);
            scratch = nullptr;
            scratchBytes = 0;
            JST_CHECK(Check(b200_malloc(B200Ctx(), need, &scratch), "AGC"));
            scratchBytes = need;
        }
        return Check(b200_agc(B200Ctx(), DevicePtr<void>(input), DevicePtr<void>(output),
                              input.dtype() == DataType::CF32 ? 1 : 0, laneCount, samples, tileSize, reference, epsilon,
                              minGain, maxGain, maxGainChange, scratch, stream), "AGC");
    }
    Result computeDeinitialize() override {
        b200_free(B200Ctx(), scratch);
        scratch = nullptr;
        scratchBytes = 0;
        return Result::SUCCESS;
    }
    void* scratch = nullptr;
    uint64_t scratchBytes = 0;
};
JST_REGISTER_MODULE(AgcImplB200, DeviceType::CUDA, RuntimeType::NATIVE, "b200");

// ---- amplitude -------------------------------------------------------------------------------------------
struct AmplitudeImplB200 : public AmplitudeImpl, public NativeCudaRuntimeContext, public Scheduler::Context {
    Result computeSubmit(const cudaStream_t& stream) override {
        if (!input.contiguous()) {
            JST_ERROR("[MODULE_AMPLITUDE_B200] Strided inputs are not supported by this provider yet.");
            return Result::ERROR;
        }
        if (input.dtype() == DataType::CF32) {
            return Check(b200_amplitude_cf32(B200Ctx(), DevicePtr<b200_cf32>(input), DevicePtr<float>(output),
                                             input.size(), scalingCoeff, stream), "AMPLITUDE");
        }
        return Check(b200_amplitude_f32(B200Ctx(), DevicePtr<float>(input), DevicePtr<float>(output), input.size(),
                                        scalingCoeff, stream), "AMPLITUDE");
    }
};
JST_REGISTER_MODULE(AmplitudeImplB200, DeviceType::CUDA, RuntimeType::NATIVE, "b200");

// ---- range -------------------------------------------------------------------------------------------------
struct RangeImplB200 : public RangeImpl, public NativeCudaRuntimeContext, public Scheduler::Context {
    Result computeSubmit(const cudaStream_t& stream) override {
        if (!input.contiguous() || input.dtype() != DataType::F32) {
            JST_ERROR("[MODULE_RANGE_B200] Only contiguous F32 inputs are supported by this provider.");
            return Result::ERROR;
        }
        return Check(b200_range_f32(B200Ctx(), DevicePtr<float>(input), DevicePtr<float>(output), input.size(),
                                    scalingCoeff, offsetCoeff, stream), "RANGE");
    }
};
JST_REGISTER_MODULE(RangeImplB200, DeviceType::CUDA, RuntimeType::NATIVE, "b200");

// ---- expand_dims (view) / multiply_constant ----------------------------------------------------------------
struct ExpandDimsImplB200 : public ExpandDimsImpl, public NativeCudaRuntimeContext, public Scheduler::Context {
    Result computeSubmit(const cudaStream_t&) override { return Result::SUCCESS; }
};
JST_REGISTER_MODULE(ExpandDimsImplB200, DeviceType::CUDA, RuntimeType::NATIVE, "b200");

struct MultiplyConstantImplB200 : public MultiplyConstantImpl, public NativeCudaRuntimeContext,
                                  public Scheduler::Context {
    Result computeSubmit(const cudaStream_t& stream) override {
        if (!input.contiguous()) {
            JST_ERROR("[MODULE_MULTIPLY_CONSTANT_B200] Strided inputs are not supported by this provider.");
            return Result::ERROR;
        }
        if (input.dtype() == DataType::CF32) {
            return Check(b200_multiply_constant_cf32(B200Ctx(), DevicePtr<b200_cf32>(input),
                                                     DevicePtr<b200_cf32>(output), input.size(), constant, stream),
                         "MULTIPLY_CONSTANT");
        }
        if (input.dtype() == DataType::F32) {
            return Check(b200_multiply_constant_f32(B200Ctx(), DevicePtr<float>(input), DevicePtr<float>(output),
                                                    input.size(), constant, stream), "MULTIPLY_CONSTANT");
        }
        JST_ERROR("[MODULE_MULTIPLY_CONSTANT_B200] Unsupported data type '{}'.", input.dtype());
        return Result::ERROR;
    }
};
JST_REGISTER_MODULE(MultiplyConstantImplB200, DeviceType::CUDA, RuntimeType::NATIVE, "b200");

// ---- filter_taps (STATIC_OUTPUT: F64 on the host with the reference's formula, uploaded once) -----------------
struct FilterTapsImplB200 : public FilterTapsImpl, public NativeCudaRuntimeContext, public Scheduler::Context {
    Result computeSubmit(const cudaStream_t& stream) override {
        const U64 heads = center.size();
        host.assign(heads * taps, b200_cf32{0.0f, 0.0f});
        JST_CHECK(Check(b200_filter_taps_host(sampleRate, bandwidth, center.data(), heads, taps, host.data()),
                        "FILTER_TAPS"));
        return Check(b200_memcpy(B200Ctx(), DevicePtr<void>(coeffs), host.data(), host.size() * sizeof(b200_cf32), 0,
                                 stream), "FILTER_TAPS");
    }
    std::vector<b200_cf32> host;     // outlives the asynchronous upload
};
JST_REGISTER_MODULE(FilterTapsImplB200, DeviceType::CUDA, RuntimeType::NATIVE, "b200");

// ---- fm -------------------------------------------------------------------------------------------------------
// validate / create (coefficients, output shape, axes) are the reference's FmImpl; the per-lane state the reference
// keeps in host vectors (previousSample, narrowDeemphasisState, stereoState) lives in the b200_fm_plan instead.
struct FmImplB200 : public FmImpl, public NativeCudaRuntimeContext, public Scheduler::Context {
    Result create() final {
        JST_CHECK(FmImpl::create());
        const Index rank = input.rank();
        if (input.dtype() != DataType::CF32 || !input.contiguous() || *signalAxes.sample + 1 != rank ||
            (signalAxes.batch && *signalAxes.batch != 0)) {
            JST_ERROR("[MODULE_FM_B200] This provider implements contiguous CF32 inputs with the sample axis innermost "
                      "and the batch axis (if any) outermost.");
            return Result::ERROR;
        }
        frameLength = input.shape(rank - 1);
        frames = signalAxes.batch ? input.shape(0) : 1;
        return Result::SUCCESS;
    }
    Result computeInitialize() override {
        const int deemphasisUs = deemphasis == "50us" ? 50 : (deemphasis == "75us" ? 75 : 0);
        return Check(b200_fm_plan_create(B200Ctx(), laneCount, sampleRate, wideBand ? 1 : 0, deemphasisUs, &plan), "FM");
    }
    Result computeSubmit(const cudaStream_t& stream) override {
        return Check(b200_fm_exec(plan, DevicePtr<b200_cf32>(input), DevicePtr<float>(output), frames, frameLength,
                                  stream), "FM");
    }
    Result computeDeinitialize() override {
        const auto result = plan ? Check(b200_fm_plan_destroy(plan), "FM") : Result::SUCCESS;
        plan = nullptr;
        return result;
    }
    b200_fm_plan* plan = nullptr;
    U64 frames = 1, frameLength = 0;
};
JST_REGISTER_MODULE(FmImplB200, DeviceType::CUDA, RuntimeType::NATIVE, "b200");

// ---- spectral_chain: the per-cycle part of spectrum_engine as ONE kernel ----------------------------------------
// Inputs: `buffer` (CF32 or complex integer, sample axis innermost) and `window` (CF32, n taps: the settled
// window -> invert [-> reshape] output). Output `buffer`: F32, the input's shape and attributes.
struct SpectralChainImplB200 : public Module::Impl, public DynamicConfig<SpectralChain>,
                               public NativeCudaRuntimeContext, public Scheduler::Context {
    Result validate() override {
        const auto& config = *candidate();
        if (!inputs().contains("buffer")) {
            return Result::SUCCESS;
        }
        const Tensor& tensor = inputs().at("buffer").tensor;
        if (!tensor.validShape() || tensor.size() == 0) {
            return Result::SUCCESS;
        }
        if (tensor.dtype() != DataType::CF32 && B200::IntegerDtypeCode(tensor.dtype()) < B200_DTYPE_CI8) {
            JST_ERROR("[MODULE_SPECTRAL_CHAIN_B200] Input must have data type CF32 or a complex integer type.");
            return Result::ERROR;
        }
        SignalAxes axes;
        if (ResolveSignalAxes(tensor, axes) != Result::SUCCESS || !axes.sample) {
            JST_ERROR("[MODULE_SPECTRAL_CHAIN_B200] Input signal axis metadata is invalid.");
            return Result::ERROR;
        }
        if (*axes.sample + 1 != tensor.rank() || !tensor.contiguous()) {
            JST_ERROR("[MODULE_SPECTRAL_CHAIN_B200] The sample axis must be the innermost axis of a contiguous tensor.");
            return Result::ERROR;
        }
        if (config.enableAgc && tensor.shape(tensor.rank() - 1) != 4096) {
            JST_ERROR("[MODULE_SPECTRAL_CHAIN_B200] The fused AGC stage exists for 4096-point spectra only; wire "
                      "fft -> agc -> amplitude for other lengths.");
            return Result::ERROR;
        }
        return Result::SUCCESS;
    }
    Result define() override {
        JST_CHECK(defineTaint(Module::Taint::STATELESS));
        JST_CHECK(defineInterfaceInput("buffer"));
        JST_CHECK(defineInterfaceInput("window"));
        return defineInterfaceOutput("buffer");
    }
    Result create() override {
        input = inputs().at("buffer").tensor;
        window = inputs().at("window").tensor;
        n = input.shape(input.rank() - 1);
        batch = input.size() / n;
        if (window.dtype() != DataType::CF32 || window.size() != n || !window.contiguous()) {
            JST_ERROR("[MODULE_SPECTRAL_CHAIN_B200] Window must be a contiguous CF32 tensor with one tap per sample.");
            return Result::ERROR;
        }
        dtypeCode = input.dtype() == DataType::CF32 ? B200_DTYPE_CF32 : B200::IntegerDtypeCode(input.dtype());
        JST_CHECK(Check(b200_amplitude_scaling_coeff(n, &amplitudeCoeff), "SPECTRAL_CHAIN"));
        JST_CHECK(Check(b200_range_coefficients(rangeMin, rangeMax, &scalingCoeff, &offsetCoeff), "SPECTRAL_CHAIN"));
        JST_CHECK(output.create(input.device(), DataType::F32, input.shape()));
        JST_CHECK(output.propagateAttributes(input));
        columnSums = Tensor();
        if (publishColumnSums && !enableAgc) {
            JST_CHECK(columnSums.create(input.device(), DataType::F32, {n}));
            JST_CHECK(output.setAttribute(B200::kColumnSumsAttribute, columnSums));
        }
        outputs()["buffer"].produced(name(), "buffer", output);
        return Result::SUCCESS;
    }
    Result reconfigure() override {     // range limits change in place, like RangeImpl::reconfigure
        const auto& config = *candidate();
        if (config.enableScale != enableScale || config.enableAgc != enableAgc ||
            config.publishColumnSums != publishColumnSums) {
            return Result::RECREATE;
        }
        rangeMin = config.rangeMin;
        rangeMax = config.rangeMax;
        agcReference = config.agcReference;
        agcEpsilon = config.agcEpsilon;
        agcMinGain = config.agcMinGain;
        agcMaxGain = config.agcMaxGain;
        return Check(b200_range_coefficients(rangeMin, rangeMax, &scalingCoeff, &offsetCoeff), "SPECTRAL_CHAIN");
    }
    Result computeSubmit(const cudaStream_t& stream) override {
        if (!plan) {
            // The window is a STATIC_OUTPUT tensor produced earlier in this first cycle on this stream: wait for it
            // once, then the plan captures it (real part only when the imaginary part is identically zero).
            if (cudaStreamSynchronize(stream) != cudaSuccess) {
                JST_ERROR("[MODULE_SPECTRAL_CHAIN_B200] Can't synchronize the stream before capturing the window.");
                return Result::ERROR;
            }
            JST_CHECK(Check(b200_chain_plan_create(B200Ctx(), n, batch, DevicePtr<b200_cf32>(window), &plan),
                            "SPECTRAL_CHAIN"));
        }
        if (enableAgc) {
            return Check(b200_chain_exec_agc(plan, DevicePtr<void>(input), dtypeCode, DevicePtr<float>(output), batch,
                                             amplitudeCoeff, enableScale ? 1 : 0, scalingCoeff, offsetCoeff,
                                             agcReference, agcEpsilon, agcMinGain, agcMaxGain, stream), "SPECTRAL_CHAIN");
        }
        if (columnSums.size() != 0) {
            return Check(b200_chain_exec_colsum(plan, DevicePtr<void>(input), dtypeCode, DevicePtr<float>(output), batch,
                                                amplitudeCoeff, enableScale ? 1 : 0, scalingCoeff, offsetCoeff,
                                                DevicePtr<float>(columnSums), stream), "SPECTRAL_CHAIN");
        }
        return Check(b200_chain_exec_typed(plan, DevicePtr<void>(input), dtypeCode, DevicePtr<float>(output), batch,
                                           amplitudeCoeff, enableScale ? 1 : 0, scalingCoeff, offsetCoeff, stream),
                     "SPECTRAL_CHAIN");
    }
    Result computeDeinitialize() override {
        const auto result = plan ? Check(b200_chain_plan_destroy(plan), "SPECTRAL_CHAIN") : Result::SUCCESS;
        plan = nullptr;
        return result;
    }
    Tensor input, window, output, columnSums;
    U64 n = 0, batch = 0;
    int dtypeCode = B200_DTYPE_CF32;
    float amplitudeCoeff = 0.0f, scalingCoeff = 0.0f, offsetCoeff = 0.0f;
    b200_chain_plan* plan = nullptr;
};
JST_REGISTER_MODULE(SpectralChainImplB200, DeviceType::CUDA, RuntimeType::NATIVE, "b200");

// ---- fir_filter: the per-cycle part of the filter block as ONE streaming (decimating, multi-head) FIR kernel ----
// Inputs: `signal` CF32 [T] or [B, T] (sample axis innermost), `coeffs` CF32 [heads, taps] (settled filter_taps
// output). Output `buffer`: [.., heads, T / R], channelAxis = the old sample axis, sampleAxis = +1 — what the
// reference block publishes (src/domains/dsp/filter/block_impl.cc:250-262,571-577).
// With a batch axis the B rows are consecutive frames of ONE stream (overlap_add carries frame k's tail into frame
// k+1, overlap_add/module_impl_native_cpu.cc:155-174); without one they are independent lanes, each with its own
// tail across cycles (:176-198) — one plan per lane here.
struct FirFilterImplB200 : public Module::Impl, public DynamicConfig<FirFilter>, public NativeCudaRuntimeContext,
                           public Scheduler::Context {
    static constexpr U64 kMaxLanes = 256;

    Result validate() override {
        const auto& config = *candidate();
        validatedAxes = {};
        if (config.decimation == 0) {
            JST_ERROR("[MODULE_FIR_FILTER_B200] Decimation must be at least 1.");
            return Result::ERROR;
        }
        if (!inputs().contains("signal")) {
            return Result::SUCCESS;
        }
        const Tensor& tensor = inputs().at("signal").tensor;
        if (!tensor.validShape() || tensor.size() == 0) {
            return Result::SUCCESS;
        }
        if (tensor.dtype() != DataType::CF32) {
            JST_ERROR("[MODULE_FIR_FILTER_B200] Signal input must be CF32.");
            return Result::ERROR;
        }
        if (ResolveSignalAxes(tensor, validatedAxes) != Result::SUCCESS || !validatedAxes.sample) {
            JST_ERROR("[BLOCK_FILTER] Signal axis metadata is invalid.");
            return Result::ERROR;
        }
        if (validatedAxes.channel) {
            JST_ERROR("[BLOCK_FILTER] Signal already has channelAxis. Generated filter channels cannot be nested.");
            return Result::ERROR;
        }
        const Index rank = tensor.rank();
        const bool layoutOk = tensor.contiguous() && *validatedAxes.sample + 1 == rank &&
                              (rank == 1 || (rank == 2 && (!validatedAxes.batch || *validatedAxes.batch == 0)));
        if (!layoutOk) {
            JST_ERROR("[MODULE_FIR_FILTER_B200] Supported layouts: contiguous [T] or [rows, T] with the sample axis "
                      "innermost.");
            return Result::ERROR;
        }
        if (tensor.shape(rank - 1) % config.decimation != 0) {
            JST_ERROR("[MODULE_FIR_FILTER_B200] Frame length must be a multiple of the decimation.");
            return Result::ERROR;
        }
        if (rank == 2 && !validatedAxes.batch && tensor.shape(0) > kMaxLanes) {
            JST_ERROR("[MODULE_FIR_FILTER_B200] At most {} independent lanes (rows without a batchAxis).", kMaxLanes);
            return Result::ERROR;
        }
        return Result::SUCCESS;
    }
    Result define() override {
        JST_CHECK(defineInterfaceInput("signal"));
        JST_CHECK(defineInterfaceInput("coeffs"));
        return defineInterfaceOutput("buffer");
    }
    Result create() override {
        input = inputs().at("signal").tensor;
        coeffs = inputs().at("coeffs").tensor;
        if (coeffs.dtype() != DataType::CF32 || coeffs.rank() != 2 || !coeffs.contiguous()) {
            JST_ERROR("[MODULE_FIR_FILTER_B200] Coefficients must be a contiguous CF32 [heads, taps] tensor.");
            return Result::ERROR;
        }
        heads = coeffs.shape(0);
        taps = coeffs.shape(1);
        const Index rank = input.rank();
        const Index sampleAxis = rank - 1;
        frameLength = input.shape(sampleAxis);
        const U64 rows = input.size() / frameLength;
        lanes = (rank == 2 && !validatedAxes.batch) ? rows : 1;
        frames = lanes > 1 ? 1 : rows;
        Shape outputShape = input.shape();
        outputShape[sampleAxis] = heads;
        outputShape.push_back(frameLength / decimation);
        JST_CHECK(output.create(input.device(), DataType::CF32, outputShape));
        JST_CHECK(output.propagateAttributes(input));
        SignalAxes outputAxes;
        outputAxes.sample = sampleAxis + 1;
        outputAxes.channel = sampleAxis;
        if (validatedAxes.batch) {
            outputAxes.batch = *validatedAxes.batch >= sampleAxis ? *validatedAxes.batch + 1 : *validatedAxes.batch;
        }
        JST_CHECK(SetSignalAxes(output, outputAxes));
        outputs()["buffer"].produced(name(), "buffer", output);
        return Result::SUCCESS;
    }
    Result createPlans(const cudaStream_t& stream) {
        // The taps are a STATIC_OUTPUT tensor uploaded earlier in this first cycle on this stream.
        std::vector<b200_cf32> host(heads * taps);
        JST_CHECK(Check(b200_memcpy(B200Ctx(), host.data(), DevicePtr<void>(coeffs), host.size() * sizeof(b200_cf32), 1,
                                    stream), "FIR_FILTER"));
        JST_CHECK(Check(b200_stream_synchronize(B200Ctx(), stream), "FIR_FILTER"));
        bool translate = false;
        std::vector<int64_t> bins(heads, 0);
        for (U64 head = 0; head < heads && head < centerBins.size(); ++head) {
            bins[head] = static_cast<int64_t>(std::llround(centerBins[head]));
            translate = translate || bins[head] != 0;
        }
        plans.assign(lanes, nullptr);
        for (auto& plan : plans) {
            JST_CHECK(Check(b200_fir_plan_create(B200Ctx(), host.data(), taps, heads, decimation, &plan), "FIR_FILTER"));
            if (translate) {
                JST_CHECK(Check(b200_fir_plan_set_translation(plan, frameLength, bins.data()), "FIR_FILTER"));
            }
        }
        return Result::SUCCESS;
    }
    Result computeSubmit(const cudaStream_t& stream) override {
        if (plans.empty()) {
            const auto result = createPlans(stream);
            if (result != Result::SUCCESS) {
                computeDeinitialize();
                return result;
            }
        }
        const auto* x = DevicePtr<b200_cf32>(input);
        auto* y = DevicePtr<b200_cf32>(output);
        const U64 outputRow = heads * (frameLength / decimation);
        for (U64 lane = 0; lane < lanes; ++lane) {
            JST_CHECK(Check(b200_fir_exec(plans[lane], x + lane * frameLength, y + lane * outputRow, frames, frameLength,
                                          stream), "FIR_FILTER"));
        }
        return Result::SUCCESS;
    }
    Result computeDeinitialize() override {
        Result result = Result::SUCCESS;
        for (auto* plan : plans) {
            if (plan && b200_fir_plan_destroy(plan) != B200_SUCCESS) {
                result = Result::ERROR;
            }
        }
        plans.clear();
        return result;
    }
    Tensor input, coeffs, output;
    SignalAxes validatedAxes;
    U64 heads = 0, taps = 0, frameLength = 0, frames = 0, lanes = 1;
    std::vector<b200_fir_plan*> plans;
};
JST_REGISTER_MODULE(FirFilterImplB200, DeviceType::CUDA, RuntimeType::NATIVE, "b200");

// ---- the separate stages of the filter wiring: pad, unpad, fold, overlap_add, phase_correction --------------------
// What the `filter` block (layouts the fused FIR does not take) and the `filter_engine` block wire between their FFTs,
// src/domains/dsp/filter/block_impl.cc:350-582. pad, unpad, fold and overlap_add are not DISCONTIGUOUS: the reference
// hands them contiguous inputs (src/module.cc:154-157), viewed here as [outer, axis, inner].
namespace {

bool RealOrComplex(const Tensor& tensor) {
    return tensor.dtype() == DataType::F32 || tensor.dtype() == DataType::CF32;
}

void AxisView(const Shape& shape, const Index axis, U64& outer, U64& inner) {
    outer = 1;
    inner = 1;
    for (Index d = 0; d < axis; ++d) outer *= shape[d];
    for (Index d = axis + 1; d < shape.size(); ++d) inner *= shape[d];
}

}  // namespace

// pad — src/domains/core/pad/module_impl_native_cpu.cc:75-142: the body is one strided copy, the zero tail a stride-0
// copy of a zeroed element (a plain memset when there is a single outer slice).
struct PadImplB200 : public PadImpl, public NativeCudaRuntimeContext, public Scheduler::Context {
    Result create() final {
        JST_CHECK(PadImpl::create());
        if (!RealOrComplex(input)) {
            JST_ERROR("[MODULE_PAD_B200] Unsupported data type '{}' (F32 and CF32 only).", input.dtype());
            return Result::ERROR;
        }
        AxisView(input.shape(), resolvedAxis, outer, inner);
        JST_CHECK(zero.create(input.device(), input.dtype(), {1}));    // zero-filled allocation
        return Result::SUCCESS;
    }
    Result computeSubmit(const cudaStream_t& stream) override {
        const int bytes = static_cast<int>(input.elementSize());
        auto* out = DevicePtr<std::uint8_t>(output);
        const U64 body = inputAxisSize * inner, row = outputAxisSize * inner, tail = size * inner;
        const U64 shape[2] = {outer, body}, src[2] = {body, 1}, dst[2] = {row, 1};
        JST_CHECK(Check(b200_copy_strided(B200Ctx(), DevicePtr<void>(input), out, bytes, 2, shape, src, dst, stream), "PAD"));
        if (tail == 0) {
            return Result::SUCCESS;
        }
        if (outer == 1) {
            return Check(b200_memset(B200Ctx(), out + body * bytes, 0, tail * bytes, stream), "PAD");
        }
        const U64 tailShape[2] = {outer, tail}, zeroStride[2] = {0, 0};
        return Check(b200_copy_strided(B200Ctx(), DevicePtr<void>(zero), out + body * bytes, bytes, 2, tailShape, zeroStride,
                                       dst, stream), "PAD");
    }
    U64 outer = 1, inner = 1;
    Tensor zero;
};
JST_REGISTER_MODULE(PadImplB200, DeviceType::CUDA, RuntimeType::NATIVE, "b200");

// unpad — src/domains/core/unpad/module_impl_native_cpu.cc:75-142: body and tail, two strided copies.
struct UnpadImplB200 : public UnpadImpl, public NativeCudaRuntimeContext, public Scheduler::Context {
    Result create() final {
        JST_CHECK(UnpadImpl::create());
        if (!RealOrComplex(input)) {
            JST_ERROR("[MODULE_UNPAD_B200] Unsupported data type '{}' (F32 and CF32 only).", input.dtype());
            return Result::ERROR;
        }
        AxisView(input.shape(), resolvedAxis, outer, inner);
        return Result::SUCCESS;
    }
    Result computeSubmit(const cudaStream_t& stream) override {
        const int bytes = static_cast<int>(input.elementSize());
        const auto* in = DevicePtr<std::uint8_t>(input);
        const U64 row = inputAxisSize * inner, body = unpadAxisSize * inner, tail = size * inner;
        if (body != 0) {
            const U64 shape[2] = {outer, body}, src[2] = {row, 1}, dst[2] = {body, 1};
            JST_CHECK(Check(b200_copy_strided(B200Ctx(), in, DevicePtr<void>(outputUnpadded), bytes, 2, shape, src, dst,
                                              stream), "UNPAD"));
        }
        if (tail != 0) {
            const U64 shape[2] = {outer, tail}, src[2] = {row, 1}, dst[2] = {tail, 1};
            JST_CHECK(Check(b200_copy_strided(B200Ctx(), in + body * bytes, DevicePtr<void>(outputPad), bytes, 2, shape, src,
                                              dst, stream), "UNPAD"));
        }
        return Result::SUCCESS;
    }
    U64 outer = 1, inner = 1;
};
JST_REGISTER_MODULE(UnpadImplB200, DeviceType::CUDA, RuntimeType::NATIVE, "b200");

// fold — b200_fold. The per-channel offsets (input attribute "channelOffsets") go to the device once, when the module
// initialises.
struct FoldImplB200 : public FoldImpl, public NativeCudaRuntimeContext, public Scheduler::Context {
    Result create() final {
        JST_CHECK(FoldImpl::create());
        if (!RealOrComplex(input)) {
            JST_ERROR("[MODULE_FOLD_B200] Unsupported input data type: {}.", input.dtype());
            return Result::ERROR;
        }
        AxisView(input.shape(), resolvedAxis, outer, inner);
        channelInner = 1;
        if (!channelOffsets.empty()) {
            for (Index d = *channelAxis + 1; d < output.rank(); ++d) channelInner *= output.shape(d);
        }
        return Result::SUCCESS;
    }
    Result computeInitialize() override {
        if (channelOffsets.empty()) {
            return Result::SUCCESS;
        }
        const U64 bytes = channelOffsets.size() * sizeof(U64);
        JST_CHECK(Check(b200_malloc(B200Ctx(), bytes, &offsetsDevice), "FOLD"));
        JST_CHECK(Check(b200_memcpy(B200Ctx(), offsetsDevice, channelOffsets.data(), bytes, 0, nullptr), "FOLD"));
        return Check(b200_stream_synchronize(B200Ctx(), nullptr), "FOLD");
    }
    Result computeSubmit(const cudaStream_t& stream) override {
        return Check(b200_fold(B200Ctx(), DevicePtr<void>(input), DevicePtr<void>(output),
                               input.dtype() == DataType::CF32 ? 1 : 0, outer, input.shape(resolvedAxis), inner, size,
                               offset, static_cast<const uint64_t*>(offsetsDevice), channelOffsets.size(), channelInner,
                               stream), "FOLD");
    }
    Result computeDeinitialize() override {
        const auto result = Check(b200_free(B200Ctx(), offsetsDevice), "FOLD");
        offsetsDevice = nullptr;
        return result;
    }
    U64 outer = 1, inner = 1, channelInner = 1;
    void* offsetsDevice = nullptr;
};
JST_REGISTER_MODULE(FoldImplB200, DeviceType::CUDA, RuntimeType::NATIVE, "b200");

// overlap_add — b200_overlap_add. previousOverlap is the reference's own module tensor, allocated on the device (zero-
// filled) and carried there. create() repeats OverlapAddImpl::create (module_impl.cc:129-151) except its host
// std::memset of that tensor, which a device allocation does not allow.
struct OverlapAddImplB200 : public OverlapAddImpl, public NativeCudaRuntimeContext, public Scheduler::Context {
    Result create() final {
        inputBuffer = validatedInputBuffer;
        inputOverlap = validatedInputOverlap;
        batchAxis = validatedBatchAxis;
        if (!RealOrComplex(inputBuffer) || inputOverlap.dtype() != inputBuffer.dtype()) {
            JST_ERROR("[MODULE_OVERLAP_ADD_B200] Buffer and overlap must both be F32 or both CF32.");
            return Result::ERROR;
        }
        JST_CHECK(output.create(inputBuffer.device(), inputBuffer.dtype(), inputBuffer.shape()));
        JST_CHECK(output.propagateAttributes(inputBuffer));
        JST_CHECK(previousOverlap.create(inputBuffer.device(), inputBuffer.dtype(), validatedPreviousOverlapShape));
        outputs()["buffer"].produced(name(), "buffer", output);

        SignalAxes axes;
        JST_CHECK(ResolveSignalAxes(inputBuffer, axes));
        sampleAxis = *axes.sample;
        AxisView(inputBuffer.shape(), sampleAxis, outer, inner);
        batches = batchAxis ? inputOverlap.shape(*batchAxis) : 1;
        batchStride = inputOverlap.size();
        if (batchAxis) {
            U64 ignored = 1;
            AxisView(inputOverlap.shape(), *batchAxis, ignored, batchStride);
        }
        return Result::SUCCESS;
    }
    Result computeSubmit(const cudaStream_t& stream) override {
        return Check(b200_overlap_add(B200Ctx(), DevicePtr<void>(inputBuffer), DevicePtr<void>(inputOverlap),
                                      DevicePtr<void>(output), DevicePtr<void>(previousOverlap),
                                      inputBuffer.dtype() == DataType::CF32 ? 1 : 0, outer, inputBuffer.shape(sampleAxis),
                                      inputOverlap.shape(sampleAxis), inner, batches, batchStride, stream),
                     "OVERLAP_ADD");
    }
    Index sampleAxis = 0;
    U64 outer = 1, inner = 1, batches = 1, batchStride = 1;
};
JST_REGISTER_MODULE(OverlapAddImplB200, DeviceType::CUDA, RuntimeType::NATIVE, "b200");

// phase_correction — b200_phase_correction. The per-channel phases advance by host arithmetic that does not depend on
// the data, kept here in F64 exactly as PhaseCorrectionImplNativeCpu keeps them (module_impl_native_cpu.cc:55-115).
// The module is DISCONTIGUOUS: a strided input is gathered into a contiguous scratch first.
struct PhaseCorrectionImplB200 : public PhaseCorrectionImpl, public NativeCudaRuntimeContext, public Scheduler::Context {
    Result create() final {
        JST_CHECK(PhaseCorrectionImpl::create());
        if (input.dtype() != DataType::CF32) {
            JST_ERROR("[MODULE_PHASE_CORRECTION_B200] Input must be CF32.");
            return Result::ERROR;
        }
        U64 ignored = 1;
        batchCount = batchAxis ? input.shape(*batchAxis) : 1;
        batchInner = 1;
        if (batchAxis) AxisView(input.shape(), *batchAxis, ignored, batchInner);
        channelCount = channelAxis ? input.shape(*channelAxis) : 1;
        channelInner = 1;
        if (channelAxis) AxisView(input.shape(), *channelAxis, ignored, channelInner);
        if (channelCount > B200_PHASE_CORRECTION_MAX_CHANNELS) {
            JST_ERROR("[MODULE_PHASE_CORRECTION_B200] {} channels exceed the supported {}.", channelCount,
                      B200_PHASE_CORRECTION_MAX_CHANNELS);
            return Result::ERROR;
        }
        phases.assign(channelCount, 0.0);
        wrappedPhaseIncrements.resize(channelCount);
        for (U64 channel = 0; channel < channelCount; ++channel) {
            const F64 increment = channelPhaseIncrements.empty() ? phaseIncrement : channelPhaseIncrements[channel];
            wrappedPhaseIncrements[channel] = std::remainder(increment, 2.0 * JST_PI);
        }
        gathered = Tensor();
        if (!input.contiguous()) {
            if (input.rank() > 8) {
                JST_ERROR("[MODULE_PHASE_CORRECTION_B200] Rank {} exceeds the supported 8.", input.rank());
                return Result::ERROR;
            }
            JST_CHECK(gathered.create(input.device(), DataType::CF32, input.shape()));
        }
        return Result::SUCCESS;
    }
    Result computeSubmit(const cudaStream_t& stream) override {
        const b200_cf32* in = DevicePtr<b200_cf32>(input);
        if (gathered.size() != 0) {
            const std::vector<U64> shape(input.shape().begin(), input.shape().end());
            const std::vector<U64> src(input.stride().begin(), input.stride().end());
            const std::vector<U64> dst(gathered.stride().begin(), gathered.stride().end());
            JST_CHECK(Check(b200_copy_strided(B200Ctx(), in, DevicePtr<b200_cf32>(gathered), 8, static_cast<int>(input.rank()),
                                              shape.data(), src.data(), dst.data(), stream), "PHASE_CORRECTION"));
            in = DevicePtr<b200_cf32>(gathered);
        }
        JST_CHECK(Check(b200_phase_correction(B200Ctx(), in, DevicePtr<b200_cf32>(output), output.size(), batchCount,
                                              batchInner, channelCount, channelInner, phases.data(),
                                              wrappedPhaseIncrements.data(), stream), "PHASE_CORRECTION"));
        for (U64 channel = 0; channel < channelCount; ++channel) {
            phases[channel] = std::remainder(
                phases[channel] + wrappedPhaseIncrements[channel] * static_cast<F64>(batchCount), 2.0 * JST_PI);
        }
        return Result::SUCCESS;
    }
    U64 batchCount = 1, batchInner = 1, channelCount = 1, channelInner = 1;
    std::vector<F64> phases, wrappedPhaseIncrements;
    Tensor gathered;
};
JST_REGISTER_MODULE(PhaseCorrectionImplB200, DeviceType::CUDA, RuntimeType::NATIVE, "b200");

// ---- lineplot / waterfall: the consumers right after the chain (SURVEY.md §8 f1) --------------------------------
// validate / create / reconfigure / present are the reference's LineplotImpl / WaterfallImpl; computeSubmit replaces
// the NVRTC kernels of lineplot/module_impl_native_cuda.cc:21-60 and waterfall/module_impl_native_cuda.cc:19-60.
struct LineplotImplB200 : public LineplotImpl, public NativeCudaRuntimeContext, public Scheduler::Context {
    Result validate() final {
        JST_CHECK(LineplotImpl::validate());
        if (inputs().contains("signal")) {
            const Tensor& tensor = inputs().at("signal").tensor;
            if (tensor.validShape() && tensor.size() != 0 && tensor.dtype() != DataType::F32) {
                JST_ERROR("[MODULE_LINEPLOT_B200] Unsupported input data type: {}.", tensor.dtype());
                return Result::ERROR;
            }
        }
        return Result::SUCCESS;
    }
    Result create() final {
        JST_CHECK(LineplotImpl::create());
        JST_CHECK(averagingBuffer.create(device(), DataType::F32, {numberOfElements}));
        uint64_t bytes = 0;
        JST_CHECK(Check(b200_lineplot_scratch_bytes(numberOfBatches, numberOfElements, decimation, &bytes), "LINEPLOT"));
        JST_CHECK(scratch.create(device(), DataType::F32, {bytes / sizeof(F32) + 1}));
        initialized = false;
        // A fused spectral_chain upstream publishes the batch sums of its output (shim/b200_provider.hh): usable when
        // the input is that module's plain row-major [batches, extent] tensor.
        columnSums = Tensor();
        if (input.hasAttribute(B200::kColumnSumsAttribute)) {
            const std::any attribute = input.attribute(B200::kColumnSumsAttribute);
            const auto* published = std::any_cast<Tensor>(&attribute);
            const U64 extent = numberOfElements * decimation;
            if (published && published->dtype() == DataType::F32 && published->size() >= extent &&
                inputElementStride == 1 && (numberOfBatches == 1 || inputBatchStride == published->size())) {
                columnSums = *published;
            }
        }
        return Result::SUCCESS;
    }
    Result presentInitialize() override { return createPresent(); }
    Result presentSubmit() override { return present(); }
    Result computeSubmit(const cudaStream_t& stream) override {
        if (numberOfElements == 0 || numberOfBatches == 0) {
            return Result::SUCCESS;
        }
        if (!initialized) {
            JST_CHECK(Check(b200_lineplot_init(B200Ctx(), DevicePtr<float>(signalPoints), DevicePtr<float>(averagingBuffer),
                                               numberOfElements, stream), "LINEPLOT"));
            initialized = true;
        }
        updateSignalPointsFlag = true;
        if (columnSums.size() != 0) {
            return Check(b200_lineplot_update_from_colsum(B200Ctx(), DevicePtr<float>(columnSums), numberOfElements,
                                                          decimation, normalizationFactor, averaging,
                                                          DevicePtr<float>(averagingBuffer), DevicePtr<float>(signalPoints),
                                                          stream), "LINEPLOT");
        }
        return Check(b200_lineplot_update(B200Ctx(), DevicePtr<float>(input), numberOfBatches, numberOfElements,
                                          inputBatchStride, inputElementStride, decimation, normalizationFactor, averaging,
                                          DevicePtr<float>(averagingBuffer), DevicePtr<float>(signalPoints),
                                          DevicePtr<void>(scratch), stream), "LINEPLOT");
    }
    Tensor averagingBuffer, scratch, columnSums;
    bool initialized = false;
};
JST_REGISTER_MODULE(LineplotImplB200, DeviceType::CUDA, RuntimeType::NATIVE, "b200");

struct WaterfallImplB200 : public WaterfallImpl, public NativeCudaRuntimeContext, public Scheduler::Context {
    Result validate() final {
        JST_CHECK(WaterfallImpl::validate());
        if (inputs().contains("signal")) {
            const Tensor& tensor = inputs().at("signal").tensor;
            if (tensor.validShape() && tensor.size() != 0 && tensor.dtype() != DataType::F32) {
                JST_ERROR("[MODULE_WATERFALL_B200] Unsupported input data type: {}.", tensor.dtype());
                return Result::ERROR;
            }
        }
        return Result::SUCCESS;
    }
    Result presentInitialize() override { return createPresent(); }
    Result presentSubmit() override { return present(); }
    Result computeSubmit(const cudaStream_t& stream) override {
        if (numberOfElements == 0 || numberOfBatches == 0) {
            return Result::SUCCESS;
        }
        JST_CHECK(Check(b200_waterfall_update(B200Ctx(), DevicePtr<float>(input), numberOfBatches, numberOfElements,
                                              inputBatchStride, inputElementStride, DevicePtr<float>(frequencyBins), height,
                                              ringState.writeIndex, stream), "WATERFALL"));
        ringState.advance(numberOfBatches, height);     // the reference's own cursor + dirty-row bookkeeping
        return Result::SUCCESS;
    }
};
JST_REGISTER_MODULE(WaterfallImplB200, DeviceType::CUDA, RuntimeType::NATIVE, "b200");

}  // namespace Jetstream::Modules
