// Block variants for provider "b200": the reference's `spectrum_engine` and `filter` blocks keep their type strings,
// config, ports, validation and per-module wiring for every other provider, and — when a flowgraph node selects
// `device: cuda / runtime: native / provider: b200` — create ONE fused module for the per-cycle part of the chain
// instead of 4-5 (spectrum_engine) or 9-11 (filter) modules.
//
// Block lookup is by type string only and duplicate registrations are an error (src/registry.cc:263-312), so a
// provider cannot ADD a second "spectrum_engine". This TU therefore REPLACES the two reference block TUs at build
// time (oracle/build_shim.sh leaves src/domains/dsp/{spectrum_engine,filter}/block_impl.cc out of the link): it
// compiles them in place, unmodified, with their static registration turned off, derives from their Impl classes
// and registers the derived classes under the reference's own requirement lists. Upstream, the same thing is a
// 10-line `if (provider() == "b200")` branch at the top of each block's create() — INTEGRATION.md §1 shows it.
#include <cmath>
#include <memory>
#include <vector>

#include <jetstream/registry.hh>

#include "b200_provider.hh"

#pragma push_macro("JST_REGISTER_BLOCK")
#undef JST_REGISTER_BLOCK
#define JST_REGISTER_BLOCK(...)
#include "domains/dsp/spectrum_engine/block_impl.cc"   // NOLINT(bugprone-suspicious-include): reference TU, in place
#include "domains/dsp/filter/block_impl.cc"            // NOLINT(bugprone-suspicious-include)
#pragma pop_macro("JST_REGISTER_BLOCK")

// Blocks this provider runs with the reference's own wiring and registration, unchanged: the filter_engine channeliser
// and the single-module blocks of a hand-wired overlap-add flowgraph (examples/flowgraphs/overlap-add-fold.yml). Their
// modules are the reference's CPU modules and the b200 modules of shim/b200_modules.cc.
#include "domains/dsp/filter_engine/block_impl.cc"     // NOLINT(bugprone-suspicious-include)
#include "domains/dsp/filter_taps/block_impl.cc"       // NOLINT(bugprone-suspicious-include)
#include "domains/dsp/fold/block_impl.cc"              // NOLINT(bugprone-suspicious-include)
#include "domains/dsp/overlap_add/block_impl.cc"       // NOLINT(bugprone-suspicious-include)
#include "domains/dsp/phase_correction/block_impl.cc"  // NOLINT(bugprone-suspicious-include)
#include "domains/core/pad/block_impl.cc"              // NOLINT(bugprone-suspicious-include)
#include "domains/core/unpad/block_impl.cc"            // NOLINT(bugprone-suspicious-include)
#include "domains/core/multiply/block_impl.cc"         // NOLINT(bugprone-suspicious-include)
#include "domains/core/expand_dims/block_impl.cc"      // NOLINT(bugprone-suspicious-include)

namespace Jetstream::Blocks {

namespace {

bool FusedTarget(const DeviceType& device, const RuntimeType& runtime, const ProviderType& provider) {
    return device == DeviceType::CUDA && runtime == RuntimeType::NATIVE && provider == "b200";
}

}  // namespace

// ---- spectrum_engine ------------------------------------------------------------------------------------------
// reference wiring: src/domains/dsp/spectrum_engine/block_impl.cc:120-217
//   cast_input -> (window -> invert -> reshape_window) -> multiply -> fft -> [agc] -> amplitude -> [range]
// b200 wiring:
//   cast_input -> (window -> invert -> reshape_window) -> spectral_chain
// The window modules stay separate STATIC_OUTPUT modules and settle after the first cycle as in the reference
// (spectrum_engine/block_tests.cc:103-122). Inputs the fused kernel does not cover (sample axis not innermost,
// AGC with a length other than 4096) take the reference wiring on this provider's per-module kernels.
struct SpectrumEngineImplB200 : public SpectrumEngineImpl {
    Result configure() override {
        JST_CHECK(SpectrumEngineImpl::configure());
        chainConfig->enableScale = enableScale;
        chainConfig->enableAgc = enableAgc;
        chainConfig->rangeMin = rangeMin;
        chainConfig->rangeMax = rangeMax;
        chainConfig->agcReference = agcConfig->reference;
        chainConfig->agcEpsilon = agcConfig->epsilon;
        chainConfig->agcMinGain = agcConfig->minGain;
        chainConfig->agcMaxGain = agcConfig->maxGain;
        return Result::SUCCESS;
    }

    Result create() override {
        if (!FusedTarget(device(), runtime(), provider()) || !candidateSampleAxis) {
            return SpectrumEngineImpl::create();
        }
        const auto& inputPort = inputs().at("buffer");
        const Tensor& inputTensor = inputPort.tensor;
        const Index axis = *candidateSampleAxis;
        const U64 size = inputTensor.shape(axis);
        if (axis + 1 != inputTensor.rank() || !inputTensor.contiguous() || (enableAgc && size != 4096)) {
            return SpectrumEngineImpl::create();
        }

        JST_CHECK(moduleCreate("cast_input", castInputConfig, {{"buffer", inputPort}}));
        const auto complexInput = moduleGetOutput({"cast_input", "buffer"});

        windowConfig->size = size;
        JST_CHECK(moduleCreate("window", windowConfig, {}));
        auto windowOutput = moduleGetOutput({"window", "window"});
        JST_CHECK(SetSignalAxes(windowOutput.tensor, {.sample = Index{0}}));
        JST_CHECK(moduleCreate("invert", invertConfig, {{"signal", windowOutput}}));

        std::string windowShape = "[";
        for (Index dimension = 0; dimension < inputTensor.rank(); ++dimension) {
            windowShape += (dimension ? ", " : "") + std::to_string(dimension == axis ? size : U64{1});
        }
        reshapeWindowConfig->shape = windowShape + "]";
        JST_CHECK(moduleCreate("reshape_window", reshapeWindowConfig,
                               {{"buffer", moduleGetOutput({"invert", "signal"})}}));
        auto reshapedWindow = moduleGetOutput({"reshape_window", "buffer"});
        JST_CHECK(SetSignalAxes(reshapedWindow.tensor, {.sample = axis}));

        JST_CHECK(moduleCreate("spectral_chain", chainConfig, {{"buffer", complexInput}, {"window", reshapedWindow}}));
        return moduleExposeOutput("buffer", {"spectral_chain", "buffer"});
    }

 protected:
    std::shared_ptr<Modules::SpectralChain> chainConfig = std::make_shared<Modules::SpectralChain>();
};

JST_REGISTER_BLOCK(SpectrumEngineImplB200,
                   {"cast"}, {"window"}, {"invert"}, {"reshape"}, {"multiply"}, {"fft"}, {"amplitude"},
                          {"agc", true}, {"range", true});

// ---- filter ---------------------------------------------------------------------------------------------------
// reference wiring: src/domains/dsp/filter/block_impl.cc:350-582 (filter_taps, cast, expand_dims, 2 x pad, 2 x fft,
// reshape, multiply, [fold], ifft, multiply_constant, [phase_correction], [unpad, overlap_add]).
// b200 wiring: filter_taps -> cast_signal -> fir_filter. The resampling decision and the per-head fold offsets are
// the reference's own CalculateCandidatePlan (block_impl.cc:40-168), called here on the same inputs.
struct FilterImplB200 : public FilterImpl {
    Result create() override {
        if (!FusedTarget(device(), runtime(), provider())) {
            return FilterImpl::create();
        }
        const auto& signalPort = inputs().at("signal");
        const Tensor& signalTensor = signalPort.tensor;
        SignalAxes axes;
        if (ResolveSignalAxes(signalTensor, axes) != Result::SUCCESS || !axes.sample) {
            JST_ERROR("[BLOCK_FILTER] Input validation plan is unavailable.");
            return Result::ERROR;
        }
        const Index signalSampleAxis = *axes.sample;
        const U64 signalSize = signalTensor.shape(signalSampleAxis);
        if (signalSampleAxis + 1 != signalTensor.rank() || signalTensor.rank() > 2 || !signalTensor.contiguous() ||
            (axes.batch && *axes.batch != 0)) {
            return FilterImpl::create();     // layouts the fused kernel does not take: reference wiring
        }
        FilterCandidatePlan plan;
        JST_CHECK(CalculateCandidatePlan(*this, signalSize, plan));

        JST_CHECK(moduleCreate("filter_taps", filterTapsConfig, {}));
        auto filterPort = moduleGetOutput({"filter_taps", "coeffs"});
        JST_CHECK(SetSignalAxes(filterPort.tensor, {.sample = Index{1}, .channel = Index{0}}));

        JST_CHECK(moduleCreate("cast_signal", castSignalConfig, {{"buffer", signalPort}}));
        const auto complexSignal = moduleGetOutput({"cast_signal", "buffer"});
        if (complexSignal.tensor.dtype() != DataType::CF32 || filterPort.tensor.dtype() != DataType::CF32) {
            JST_ERROR("[BLOCK_FILTER] Internal convolution inputs must be CF32.");
            return Result::ERROR;
        }

        firConfig->decimation = 1;
        firConfig->centerBins.clear();
        if (plan.resample) {
            firConfig->decimation = plan.convolutionSize / plan.resamplerSize;
            // fold offset o = (-centerBin) mod M (block_impl.cc:136-160)  ->  signed centre bin of the head
            const U64 m = plan.convolutionSize;
            for (const U64 offset : plan.resamplerOffsets) {
                const I64 bin = offset == 0 ? 0 : (offset > m / 2 ? static_cast<I64>(m - offset)
                                                                  : -static_cast<I64>(offset));
                firConfig->centerBins.push_back(static_cast<F64>(bin));
            }
        }
        JST_CHECK(moduleCreate("fir", firConfig, {{"signal", complexSignal}, {"coeffs", filterPort}}));
        JST_CHECK(moduleExposeOutput("buffer", {"fir", "buffer"}));
        if (plan.resample) {
            JST_CHECK(outputs().at("buffer").tensor.setAttribute("sampleRate", plan.resampledSampleRate));
        }
        return Result::SUCCESS;
    }

 protected:
    std::shared_ptr<Modules::FirFilter> firConfig = std::make_shared<Modules::FirFilter>();
};

JST_REGISTER_BLOCK(FilterImplB200,
                   {"filter_taps"}, {"cast"}, {"expand_dims"}, {"pad"}, {"fft"}, {"reshape"}, {"multiply"},
                          {"multiply_constant"}, {"phase_correction", true}, {"unpad", true}, {"overlap_add", true},
                          {"fold", true});

}  // namespace Jetstream::Blocks
