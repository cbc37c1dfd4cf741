// TEST INFRASTRUCTURE ONLY -- the undistortion entry points of a CPU stand-in for libb200match.so, compiled together
// with mock_b200match.cpp into a test's temporary directory, so that undistort_images runs through the host module
// (options, items, run-time symbol lookup, the C structs, the chunked pipeline) without a GPU.  Cameras are the
// library's own (csrc/undistort_camera.h).  "Undistorting" makes an image of the undistorted size: pixels filled with
// the call's running item number, or for JPEG output the bytes "MOCKJPEG <width> <height>".  Every call and item is
// appended to the file named by B2M_MOCK_UNDISTORT_LOG.
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/b200match.h"
#include "../../pycolmap_b200/csrc/undistort_camera.h"

struct b2m_undistorted {
  std::vector<b2m_camera> camera;
  std::vector<std::vector<uint8_t>> data;
};

namespace {
int g_items = 0;

void Log(const char* fmt, ...) __attribute__((format(printf, 1, 2)));
void Log(const char* fmt, ...) {
  const char* path = getenv("B2M_MOCK_UNDISTORT_LOG");
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

void b2m_undistort_opts_default(b2m_undistort_opts* o) {
  std::memset(o, 0, sizeof(*o));
  o->struct_size = sizeof(*o);
  o->max_image_size = -1;
  o->min_scale = 0.2;
  o->max_scale = 2.0;
  o->roi_max_x = o->roi_max_y = 1.0;
}

int b2m_undistort_camera(b2m_ctx*, const b2m_undistort_opts* o, const b2m_camera* c, b2m_camera* out) {
  if (!o || !c || !out || b2m::undistort::opts_problem(*o)) return B2M_EINVAL;
  b2m::undistort::undistort_camera(*o, *c, out);
  return B2M_OK;
}

int b2m_undistort_images(b2m_ctx*, const b2m_undistort_item* items, int32_t n, const b2m_undistort_opts* o,
                         b2m_undistorted** out) {
  if (!o || o->struct_size != sizeof(*o) || b2m::undistort::opts_problem(*o)) return B2M_EINVAL;
  Log("CALL %d\n", n);
  auto* R = new b2m_undistorted();
  for (int i = 0; i < n; ++i) {
    const b2m_undistort_item& it = items[i];
    if (it.struct_size != sizeof(it)) {
      delete R;
      return B2M_EINVAL;
    }
    b2m_camera u;
    b2m::undistort::undistort_camera(*o, it.camera, &u);
    Log("ITEM output=%d model=%d camera=%dx%d source=%d bytes=%lld\n", it.output, it.camera.model, it.camera.width,
        it.camera.height, it.source.kind, static_cast<long long>(it.source.kind == B2M_SOURCE_JPEG ? it.source.size :
                                                                 it.source.stride * it.source.height));
    std::vector<uint8_t> d;
    if (it.output == B2M_UNDISTORT_JPEG) {
      const std::string s = "MOCKJPEG " + std::to_string(u.width) + " " + std::to_string(u.height);
      d.assign(s.begin(), s.end());
    } else {
      d.assign(3 * static_cast<size_t>(u.width) * u.height, static_cast<uint8_t>(g_items));
    }
    ++g_items;
    R->camera.push_back(u);
    R->data.push_back(std::move(d));
  }
  *out = R;
  return B2M_OK;
}

int b2m_undistorted_get(const b2m_undistorted* r, int32_t k, b2m_undistorted_view* v) {
  if (!r || !v || k < 0 || k >= static_cast<int32_t>(r->camera.size())) return B2M_EINVAL;
  v->struct_size = sizeof(*v);
  v->status = B2M_OK;
  v->error = "";
  v->width = r->camera[k].width;
  v->height = r->camera[k].height;
  v->camera = r->camera[k];
  v->size = static_cast<int64_t>(r->data[k].size());
  v->data = r->data[k].data();
  return B2M_OK;
}

void b2m_undistorted_free(b2m_undistorted* r) { delete r; }

}  // extern "C"
