// TEST INFRASTRUCTURE ONLY -- the PatchMatch entry points of a CPU stand-in for libb200match.so, compiled together with
// mock_b200match.cpp into a test's temporary directory, so that patch_match_stereo runs through the host module (option
// and problem conversion, run-time symbol lookup, the C structs) without a GPU.  "Decoding" takes the host pixels' first
// channel; the maps of a problem are depth = depth_min + image_id everywhere and normal = (0, 0, -1).  Every image set
// and batch is appended to the file named by B2M_MOCK_PM_LOG.
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../include/b200match.h"

struct b2m_depth_maps {
  std::vector<int32_t> width, height;
  std::vector<std::vector<float>> depth, normal;
};

namespace {
std::vector<int32_t> g_w, g_h;
std::vector<int> g_has_dmap;

void Log(const char* fmt, ...) __attribute__((format(printf, 1, 2)));
void Log(const char* fmt, ...) {
  const char* path = getenv("B2M_MOCK_PM_LOG");
  if (!path) return;
  if (FILE* f = fopen(path, "a")) {
    va_list ap;
    va_start(ap, fmt);
    vfprintf(f, fmt, ap);
    va_end(ap);
    fclose(f);
  }
}
}  // namespace

extern "C" {

int b2m_debug_decode_grey(b2m_ctx*, const b2m_image_source* s, int32_t, uint8_t* grey, int32_t* width, int32_t* height) {
  if (!s || s->kind != B2M_SOURCE_PIXELS) return B2M_EINVAL;
  *width = s->width;
  *height = s->height;
  if (grey)
    for (int y = 0; y < s->height; ++y)
      for (int x = 0; x < s->width; ++x) grey[y * s->width + x] = s->data[y * s->stride + x * s->channels];
  return B2M_OK;
}

int b2m_patch_match_set_images(b2m_ctx*, int32_t n, const b2m_image* images, const double* cameras,
                               const float* const* depth_maps) {
  g_w.assign(n, 0);
  g_h.assign(n, 0);
  g_has_dmap.assign(n, 0);
  Log("SET %d", n);
  for (int i = 0; i < n; ++i) {
    g_w[i] = images[i].width;
    g_h[i] = images[i].height;
    g_has_dmap[i] = depth_maps && depth_maps[i];
    Log(" %dx%d:%d:%.6g", g_w[i], g_h[i], g_has_dmap[i], cameras[16 * i]);
  }
  Log("\n");
  return B2M_OK;
}

int b2m_patch_match_batch(b2m_ctx*, const b2m_patch_match_problem* p, int32_t n, const b2m_patch_match_opts* o,
                          b2m_depth_maps** out) {
  if (!o || o->struct_size != sizeof(*o)) return B2M_EINVAL;
  Log("BATCH %d geom=%d filter=%d iters=%d radius=%d\n", n, o->geom_consistency, o->filter, o->num_iterations,
      o->window_radius);
  auto* M = new b2m_depth_maps();
  for (int k = 0; k < n; ++k) {
    if (p[k].struct_size != sizeof(p[k])) {
      delete M;
      return B2M_EINVAL;
    }
    const int W = g_w[p[k].ref], H = g_h[p[k].ref];
    Log("PROBLEM ref=%d id=%d n_src=%d init=%d range=%.4g,%.4g\n", p[k].ref, p[k].image_id, p[k].n_src,
        p[k].init_depth != nullptr, p[k].depth_min, p[k].depth_max);
    M->width.push_back(W);
    M->height.push_back(H);
    M->depth.emplace_back(static_cast<size_t>(W) * H, p[k].depth_min + p[k].image_id);
    std::vector<float> nrm(static_cast<size_t>(W) * H * 3, 0.f);
    for (size_t i = 2; i < nrm.size(); i += 3) nrm[i] = -1.f;
    M->normal.push_back(std::move(nrm));
  }
  *out = M;
  return B2M_OK;
}

int b2m_depth_maps_get(const b2m_depth_maps* m, int32_t k, b2m_depth_map_view* v) {
  if (!m || !v || k < 0 || k >= static_cast<int32_t>(m->width.size())) return B2M_EINVAL;
  v->struct_size = sizeof(*v);
  v->width = m->width[k];
  v->height = m->height[k];
  v->depth = m->depth[k].data();
  v->normal = m->normal[k].data();
  return B2M_OK;
}

void b2m_depth_maps_free(b2m_depth_maps* m) { delete m; }

}  // extern "C"
