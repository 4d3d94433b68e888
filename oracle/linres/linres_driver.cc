// C-ABI driver over the reference runtime's LinearResample, constructed as Audio::WavResample constructs it (audio.cpp:300-325:
// cutoff 0.99 * 0.5 * min rate as a float, 6 zeros).  The driver reads the object's phase tables and output count, which the class
// keeps private, so it opens the class's private section for this translation unit only.
#include <cstdint>
#include <cstring>
#include <vector>
#define private public
#include "resample.h"
#undef private

using funasr::LinearResample;

extern "C" {

void* linres_new(int32_t in_rate, int32_t out_rate) {
  float min_freq = in_rate < out_rate ? in_rate : out_rate;
  float cutoff = 0.99 * 0.5 * min_freq;
  return new LinearResample(in_rate, out_rate, cutoff, 6);
}

void linres_free(void* r) { delete static_cast<LinearResample*>(r); }

void linres_units(void* r, int32_t* in_unit, int32_t* out_unit) {
  LinearResample* l = static_cast<LinearResample*>(r);
  *in_unit = l->input_samples_in_unit_;
  *out_unit = l->output_samples_in_unit_;
}

// phase p: first input index, its weights into w (up to cap), returns the weight count
int32_t linres_row(void* r, int32_t p, int32_t* first, float* w, int32_t cap) {
  LinearResample* l = static_cast<LinearResample*>(r);
  *first = l->first_index_[p];
  const std::vector<float>& row = l->weights_[p];
  const int32_t n = (int32_t)row.size();
  if (w) memcpy(w, row.data(), sizeof(float) * (n < cap ? n : cap));
  return n;
}

int64_t linres_out_len(void* r, int64_t n) { return static_cast<LinearResample*>(r)->GetNumOutputSamples(n, true); }

// Resample(x, n, flush = true) into y (up to cap); returns the output count
int64_t linres_resample(void* r, const float* x, int32_t n, float* y, int64_t cap) {
  std::vector<float> out;
  static_cast<LinearResample*>(r)->Resample(x, n, true, &out);
  const int64_t k = (int64_t)out.size();
  if (y) memcpy(y, out.data(), sizeof(float) * (k < cap ? k : cap));
  return k;
}

}
