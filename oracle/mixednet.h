/* oracle/mixednet.h -- CPU ORACLE (test infrastructure only; see mixednet.c header). */
#ifndef MWWO_MIXEDNET_H_
#define MWWO_MIXEDNET_H_

#include <stddef.h>
#include <stdint.h>
#include <stdio.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct mwwo_mixednet mwwo_mixednet;

/* blob = MWW container bytes (copied).  NULL on a malformed / incomplete container, or on an architecture outside what the
 * per-step buffers hold: 1..8 blocks, 1..4 MixConv groups per block, 1..512 channels per layer, 1..64 taps per kernel,
 * 1..64 head rows, 1 <= stride <= first_conv_kernel_size. */
mwwo_mixednet *mwwo_mixednet_create(const void *blob, size_t n);
void mwwo_mixednet_free(mwwo_mixednet *m);
void mwwo_mixednet_reset(mwwo_mixednet *m);
int mwwo_mixednet_is_quantized(const mwwo_mixednet *m);
int mwwo_mixednet_stride(const mwwo_mixednet *m);
float mwwo_mixednet_input_scale(const mwwo_mixednet *m);
int mwwo_mixednet_input_zero_point(const mwwo_mixednet *m);

/* one invoke: x = [stride][40]; returns the probability (fp32) / the uint8 output value (int8) */
float mwwo_mixednet_step_f32(mwwo_mixednet *m, const float *x, float *logit_out);
int mwwo_mixednet_step_int8(mwwo_mixednet *m, const int8_t *x, int *logit_out);

/* Model.predict_spectrogram over uint16 features (stride == input_feature_slices); returns #probs */
size_t mwwo_mixednet_predict_u16(mwwo_mixednet *m, const uint16_t *feat, size_t rows, float *probs, size_t max_probs);

#ifdef __cplusplus
}
#endif
#endif
