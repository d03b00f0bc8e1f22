// mww_container.h -- a model container (microwakeword_b200/model_file.py) read into the weights one NN model runs on.
//
// Host only, no CUDA runtime calls: mww_create uploads what this produces, and tests/test_container.py builds it with g++ to
// check every refusal without a device.
#pragma once

#include <stddef.h>
#include <stdint.h>

#include <string>
#include <vector>

#include "mww_nn_generic.cuh"
#include "mww_nn_tc_prep.h"

namespace mww {

// the kernel family a model runs on.  Compiled: the okay_nabu kernels (mww_nn.cu, mww_nn_tc.cu, mww_nn_int8.cu and the live-step
// kernels); generic: the run-time-geometry kernels (mww_nn_generic.cuh); hybrid: fp32 graph with int8-weight ops, any architecture
enum class ModelKind { kCompiledF32, kCompiledI8, kGenericF32, kGenericI8, kHybrid };

// okay_nabu's geometry: what a frontend-only handle reports
const GenArch &okay_nabu_arch();

struct ModelWeights {
    ModelKind kind = ModelKind::kCompiledF32;
    GenArch G{};                    // stride, pending rows, ring state and MACs per step of every kind
    GenWeightsF32 GW{};             // fp32 tensors (fp32, hybrid and compiled fp32 models)
    GenWeightsI8 GQ{};              // int8 tensors (int8 and compiled int8 models)
    GenHybrid GH{};
    NnWeightsF32 W{};               // compiled fp32: the same tensors as GW
    TcWeights TW{};                 // compiled fp32: pre-split weights for the wgmma clip kernel (mww_nn_tc.cu)
    NnWeightsI8 Wq{};               // compiled int8: the same tensors as GQ, and the tensor-core operands
    bool tc_f16 = false;            // the first conv's weights admit fp16 hi / lo operands (tc_f16_scales) and MWW_TC_TF32 is unset
    float in_scale = 0.f, out_scale = 0.f;
    int in_zp = 0, out_zp = 0;
    // every tensor and derived operand, each at a 256-byte-aligned offset.  Until rebase() the weight pointers above that
    // point into the arena hold those offsets; `fixups` are the byte offsets of these pointers within *this.
    std::vector<unsigned char> arena;
    std::vector<size_t> fixups;

    bool quantized() const { return kind == ModelKind::kCompiledI8 || kind == ModelKind::kGenericI8; }
    bool compiled() const { return kind == ModelKind::kCompiledF32 || kind == ModelKind::kCompiledI8; }
    // the arena now lives at `base`: offsets become pointers, the compiled kinds' W / Wq take GW's / GQ's tensors, and the
    // host arena is released
    void rebase(const void *base);
};

// MWW_OK, or MWW_EMODEL / MWW_EUNSUPPORTED with the message mww_last_error reports.  Reads MWW_FORCE_GENERIC, MWW_TC_TF32 and
// MWW_NO_QLUT.
int parse_container(const uint8_t *blob, size_t n, ModelWeights *out, std::string *err);

}  // namespace mww
