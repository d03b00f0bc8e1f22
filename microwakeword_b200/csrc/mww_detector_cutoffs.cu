// mww_detector_cutoffs.cu -- the streaming detectors in per-row mode (mww_set_detector_cutoffs,
// mww_set_multi_detector_cutoffs): the plain detector's update kernel in both forms with each row's cutoff
// (mww_detector.cuh) and the models detector's over per-row descriptors (mww_detector_models.cuh).  A companion library of
// its own, so that libmww_detector.so and libmww_detector_models.so keep exactly the kernels uniform mode runs.
#include "mww_detector.cuh"
#include "mww_detector_models.cuh"

namespace mww {

cudaError_t launch_detector_update_cutoffs(const DetectorArgs &a, const double *row_cutoff, const float *probs, int n_steps, long long pitch,
                                           cudaStream_t st) {
    return launch_update_form<true>(a, row_cutoff, probs, n_steps, pitch, st);
}

cudaError_t launch_detector_models_update_cutoffs(const DetectModelsArgsT<DetectModelRows> &a, cudaStream_t st) {
    return launch_models_update_form(a, st);
}

}  // namespace mww
