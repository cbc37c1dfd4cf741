// TEST INFRASTRUCTURE ONLY -- the extraction entry points of a CPU stand-in for libb200match.so, compiled together
// with mock_b200match.cpp into a test's temporary directory, so that the host pipeline of extract_features (file
// list, cameras, batches, skips, writes) runs end to end without a GPU.  "Decoding" reads the JPEG frame header (or
// takes the pixel size); a file containing the bytes MOCKBAD does not decode, one containing MOCKSIZE decodes one
// pixel wider than its header says.  Features are a deterministic function of the decoded size that tests recompute.
// The options of every call are appended to the file named by B2M_MOCK_EXTRACT_LOG.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/b200match.h"

struct b2m_features {
  std::vector<int64_t> off{0};
  std::vector<float> kpts;
  std::vector<uint8_t> desc;
  std::vector<int32_t> width, height, status;
  std::vector<std::string> error;
};

namespace {
bool Contains(const uint8_t* p, int64_t n, const char* what) {
  const size_t k = strlen(what);
  for (int64_t i = 0; i + static_cast<int64_t>(k) <= n; ++i)
    if (memcmp(p + i, what, k) == 0) return true;
  return false;
}

bool JpegSize(const uint8_t* b, int64_t n, int* w, int* h) {
  for (int64_t i = 2; i + 9 < n;) {
    if (b[i] != 0xFF) return false;
    const int m = b[i + 1];
    const int len = (b[i + 2] << 8) | b[i + 3];
    if (m >= 0xC0 && m <= 0xCF && m != 0xC4 && m != 0xC8 && m != 0xCC) {
      *h = (b[i + 5] << 8) | b[i + 6];
      *w = (b[i + 7] << 8) | b[i + 8];
      return true;
    }
    i += 2 + len;
  }
  return false;
}
}  // namespace

extern "C" {

int b2m_extract_features_sources(b2m_ctx*, const b2m_image_source* sources, int32_t n, const b2m_extract_opts* opts,
                                 b2m_features** out) {
  if (const char* log = getenv("B2M_MOCK_EXTRACT_LOG")) {
    if (FILE* f = fopen(log, "a")) {
      fprintf(f, "%d %d %.17g %d %d\n", n, opts->first_octave, opts->peak_threshold, opts->max_image_size,
              opts->max_num_features);
      fclose(f);
    }
  }
  b2m_features* F = new b2m_features();
  for (int32_t i = 0; i < n; ++i) {
    const b2m_image_source& s = sources[i];
    int w = s.width, h = s.height;
    const int64_t bytes = s.kind == B2M_SOURCE_JPEG ? s.size : s.stride * s.height;
    bool ok = s.kind != B2M_SOURCE_JPEG || JpegSize(s.data, s.size, &w, &h);
    if (Contains(s.data, bytes, "MOCKBAD")) ok = false;
    if (Contains(s.data, bytes, "MOCKSIZE")) w += 1;
    F->width.push_back(w);
    F->height.push_back(h);
    F->status.push_back(ok ? B2M_OK : B2M_EINVAL);
    F->error.push_back(ok ? "" : "mock: does not decode");
    const int nf = ok ? 1 + (w + h) % 4 : 0;
    for (int k = 0; k < nf; ++k) {
      const float kp[6] = {k + 0.5f, w / 2.0f, 1.0f, 0.0f, 0.0f, 1.0f};
      F->kpts.insert(F->kpts.end(), kp, kp + 6);
      for (int d = 0; d < 128; ++d) F->desc.push_back(static_cast<uint8_t>((w * 7 + k + d) & 255));
    }
    F->off.push_back(F->off.back() + nf);
  }
  *out = F;
  return B2M_OK;
}

int b2m_source_features_get(const b2m_features* f, int32_t i, b2m_source_view* v) {
  if (!f || !v || i < 0 || i >= static_cast<int32_t>(f->status.size())) return B2M_EINVAL;
  v->struct_size = sizeof(*v);
  v->status = f->status[i];
  v->error = f->error[i].c_str();
  v->width = f->width[i];
  v->height = f->height[i];
  v->n = f->off[i + 1] - f->off[i];
  v->keypoints = f->kpts.data() + 6 * f->off[i];
  v->descriptors = f->desc.data() + 128 * f->off[i];
  return B2M_OK;
}

void b2m_features_free(b2m_features* f) { delete f; }

}  // extern "C"
