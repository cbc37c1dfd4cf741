#include "image_reader.h"

#include <dlfcn.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <filesystem>
#include <fstream>
#include <iterator>
#include <stdexcept>

namespace b2mh {
namespace {

const char* const kModelNames[] = {"SIMPLE_PINHOLE", "PINHOLE", "SIMPLE_RADIAL", "RADIAL", "OPENCV", "OPENCV_FISHEYE",
                                   "FULL_OPENCV", "FOV", "SIMPLE_RADIAL_FISHEYE", "RADIAL_FISHEYE", "THIN_PRISM_FISHEYE"};
const int kNumParams[] = {3, 4, 4, 5, 8, 8, 12, 5, 4, 5, 12};
bool SingleFocal(int m) { return m == 0 || m == 2 || m == 3 || m == 8 || m == 9; }

// CSVToVector<double>: split on ',' / ';', trim, skip empty fields; a field that is not a number empties the list
std::vector<double> CsvToDoubles(const std::string& csv) {
  std::vector<double> v;
  std::string field;
  auto flush = [&](std::string f) -> bool {
    const size_t a = f.find_first_not_of(" \t\r\n"), b = f.find_last_not_of(" \t\r\n");
    if (a == std::string::npos) return true;
    f = f.substr(a, b - a + 1);
    try {
      v.push_back(std::stod(f));
    } catch (const std::exception&) {
      return false;
    }
    return true;
  };
  for (char c : csv) {
    if (c == ',' || c == ';') {
      if (!flush(field)) return {};
      field.clear();
    } else {
      field.push_back(c);
    }
  }
  if (!flush(field)) return {};
  return v;
}

// ---- zlib, bound at run time like SQLite (sqlite_dyn.cc): the product links no compression library ----------------
struct Zlib {
  int (*uncompress)(unsigned char*, unsigned long*, const unsigned char*, unsigned long) = nullptr;
  unsigned long (*crc32)(unsigned long, const unsigned char*, unsigned int) = nullptr;
  unsigned long (*compress_bound)(unsigned long) = nullptr;
  int (*compress2)(unsigned char*, unsigned long*, const unsigned char*, unsigned long, int) = nullptr;
};

const Zlib& zlib() {
  static const Zlib z = [] {
    Zlib r;
    void* lib = nullptr;
    for (const char* name : {"libz.so.1", "libz.so"}) {
      lib = dlopen(name, RTLD_NOW | RTLD_LOCAL);
      if (lib) break;
    }
    if (!lib) throw std::runtime_error("[image_reader.cc] cannot load libz.so.1 (needed to decode PNG files)");
    r.uncompress = reinterpret_cast<decltype(r.uncompress)>(dlsym(lib, "uncompress"));
    r.crc32 = reinterpret_cast<decltype(r.crc32)>(dlsym(lib, "crc32"));
    r.compress_bound = reinterpret_cast<decltype(r.compress_bound)>(dlsym(lib, "compressBound"));
    r.compress2 = reinterpret_cast<decltype(r.compress2)>(dlsym(lib, "compress2"));
    if (!r.uncompress || !r.crc32 || !r.compress_bound || !r.compress2)
      throw std::runtime_error("[image_reader.cc] libz.so.1 lacks uncompress / crc32 / compressBound / compress2");
    return r;
  }();
  return z;
}

uint32_t Be32(const uint8_t* p) { return (uint32_t(p[0]) << 24) | (uint32_t(p[1]) << 16) | (uint32_t(p[2]) << 8) | p[3]; }
uint16_t Be16(const uint8_t* p) { return static_cast<uint16_t>((p[0] << 8) | p[1]); }

const uint8_t kPngMagic[8] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1a, '\n'};

ImageFormat Sniff(const std::vector<uint8_t>& b) {
  if (b.size() >= 3 && b[0] == 0xFF && b[1] == 0xD8 && b[2] == 0xFF) return ImageFormat::JPEG;
  if (b.size() >= 8 && std::memcmp(b.data(), kPngMagic, 8) == 0) return ImageFormat::PNG;
  return ImageFormat::UNKNOWN;
}

// ---- EXIF (TIFF structure inside the APP1 segment) ----------------------------------------------------------------
struct Tiff {
  const uint8_t* p;
  size_t n;
  bool le;
  bool ok(size_t off, size_t len) const { return off <= n && len <= n - off; }
  uint16_t u16(size_t o) const { return le ? static_cast<uint16_t>(p[o] | (p[o + 1] << 8)) : Be16(p + o); }
  uint32_t u32(size_t o) const {
    return le ? (uint32_t(p[o]) | (uint32_t(p[o + 1]) << 8) | (uint32_t(p[o + 2]) << 16) | (uint32_t(p[o + 3]) << 24)) : Be32(p + o);
  }
};

struct ExifTags {
  bool f35 = false, focal = false, pxdim = false, xres = false, unit = false;
  uint32_t f35_v = 0, pxdim_v = 0, unit_v = 0;
  uint32_t focal_num = 0, focal_den = 0, xres_num = 0, xres_den = 0;
};

// Reads the entries of the IFD at `off`; *exif_ifd = the Exif IFD pointer (tag 0x8769) when present.
void ReadIfd(const Tiff& t, size_t off, ExifTags* tags, uint32_t* exif_ifd) {
  if (!t.ok(off, 2)) return;
  const int count = t.u16(off);
  for (int i = 0; i < count; ++i) {
    const size_t e = off + 2 + 12 * static_cast<size_t>(i);
    if (!t.ok(e, 12)) return;
    const uint16_t tag = t.u16(e), type = t.u16(e + 2);
    const uint32_t cnt = t.u32(e + 4);
    auto scalar = [&](uint32_t* v) -> bool {  // SHORT or LONG, first value
      if (cnt < 1) return false;
      if (type == 3) *v = t.u16(e + 8);
      else if (type == 4) *v = t.u32(e + 8);
      else return false;
      return true;
    };
    auto rational = [&](uint32_t* num, uint32_t* den) -> bool {  // RATIONAL, stored at an offset
      if (type != 5 || cnt < 1) return false;
      const size_t o = t.u32(e + 8);
      if (!t.ok(o, 8)) return false;
      *num = t.u32(o);
      *den = t.u32(o + 4);
      return true;
    };
    switch (tag) {
      case 0x8769: if (exif_ifd) scalar(exif_ifd); break;
      case 0xA405: tags->f35 = scalar(&tags->f35_v); break;
      case 0x920A: tags->focal = rational(&tags->focal_num, &tags->focal_den); break;
      case 0xA002: tags->pxdim = scalar(&tags->pxdim_v); break;
      case 0xA20E: tags->xres = rational(&tags->xres_num, &tags->xres_den); break;
      case 0xA210: tags->unit = scalar(&tags->unit_v); break;
      default: break;
    }
  }
}

bool FindExif(const uint8_t* data, size_t size, ExifTags* tags) {
  size_t i = 2;  // after SOI
  while (i + 4 <= size && data[i] == 0xFF) {
    const uint8_t marker = data[i + 1];
    if (marker == 0xD8 || (marker >= 0xD0 && marker <= 0xD7) || marker == 0x01) {
      i += 2;
      continue;
    }
    if (marker == 0xDA || marker == 0xD9) break;  // start of scan: no metadata after it
    const size_t len = Be16(data + i + 2);
    if (len < 2 || i + 2 + len > size) break;
    const uint8_t* seg = data + i + 4;
    if (marker == 0xE1 && len >= 2 + 6 + 8 && std::memcmp(seg, "Exif\0\0", 6) == 0) {
      const Tiff t{seg + 6, len - 2 - 6, seg[6] == 'I'};
      if ((seg[6] == 'I' || seg[6] == 'M') && t.u16(2) == 42) {
        uint32_t exif_ifd = 0;
        ReadIfd(t, t.u32(4), tags, &exif_ifd);
        if (exif_ifd) ReadIfd(t, exif_ifd, tags, nullptr);
        return true;
      }
    }
    i += 2 + len;
  }
  return false;
}

bool JpegHeader(const std::vector<uint8_t>& b, ImageHeader* h) {
  size_t i = 2;
  while (i + 4 <= b.size()) {
    if (b[i] != 0xFF) return false;
    const uint8_t m = b[i + 1];
    if (m == 0xFF) {
      ++i;
      continue;
    }
    if (m == 0xD8 || (m >= 0xD0 && m <= 0xD7) || m == 0x01) {
      i += 2;
      continue;
    }
    const size_t len = Be16(b.data() + i + 2);
    if (len < 2 || i + 2 + len > b.size()) return false;
    // SOF0..SOF15 except DHT (C4), JPG (C8) and DAC (CC)
    if (m >= 0xC0 && m <= 0xCF && m != 0xC4 && m != 0xC8 && m != 0xCC) {
      if (len < 8) return false;
      h->height = Be16(b.data() + i + 5);
      h->width = Be16(b.data() + i + 7);
      return h->width > 0 && h->height > 0;
    }
    if (m == 0xDA || m == 0xD9) return false;
    i += 2 + len;
  }
  return false;
}

}  // namespace

int CameraModelId(const std::string& name) {
  for (int i = 0; i < 11; ++i)
    if (name == kModelNames[i]) return i;
  return -1;
}

bool VerifyCameraParams(const std::string& model, const std::string& params) {
  const int id = CameraModelId(model);
  if (id < 0) return false;
  const std::vector<double> p = CsvToDoubles(params);
  return p.empty() || static_cast<int>(p.size()) == kNumParams[id];
}

std::vector<double> InitialCameraParams(int model, double focal, int64_t width, int64_t height) {
  std::vector<double> p(kNumParams[model], 0.0);
  const int pp = SingleFocal(model) ? 1 : 2;
  for (int k = 0; k < pp; ++k) p[k] = focal;
  p[pp] = width / 2.0;
  p[pp + 1] = height / 2.0;
  if (model == 7) p[4] = 1e-2;  // FOV: omega
  return p;
}

std::vector<uint8_t> ReadFileBytes(const std::string& path) {
  std::ifstream f(path, std::ios::binary);
  if (!f) return {};
  return std::vector<uint8_t>(std::istreambuf_iterator<char>(f), std::istreambuf_iterator<char>());
}

// Bitmap::ExifFocalLength.  FreeImage hands the tags over as strings and COLMAP parses numbers back out of them, so the
// values are those strings' values: FocalLengthIn35mmFilm "%hu mm"; FocalLength "%.1f mm" (rounded to 0.1 mm);
// FocalPlaneXResolution as FIRational::toString, "num/den", or a bare integer (which the "x/y" pattern then rejects);
// FocalPlaneResolutionUnit "inches" (2) or "cm" (3).  The camera-sensor database lookup by Make / Model is not restated.
bool ExifFocalLength(const uint8_t* data, size_t size, double max_size, double* focal) {
  ExifTags t;
  if (!FindExif(data, size, &t)) return false;
  if (t.f35 && t.f35_v > 0) {
    *focal = static_cast<double>(t.f35_v) / 35.0 * max_size;
    return true;
  }
  if (!t.focal || t.focal_den == 0) return false;
  char buf[64];
  snprintf(buf, sizeof(buf), "%.1f", static_cast<double>(t.focal_num) / t.focal_den);
  const double focal_mm = std::strtod(buf, nullptr);
  if (!(t.pxdim && t.xres && t.unit) || t.xres_den == 0 || t.xres_num == 0) return false;
  if (t.xres_num % t.xres_den == 0) return false;  // printed as an integer: no "x/y" to parse
  const double x_res = static_cast<double>(static_cast<long double>(t.xres_den) / static_cast<long double>(t.xres_num));
  const double ccd_width = x_res * static_cast<double>(t.pxdim_v);
  if (!(ccd_width > 0 && focal_mm > 0)) return false;
  if (t.unit_v == 3) {
    *focal = focal_mm / (ccd_width * 10.0) * max_size;
    return true;
  }
  if (t.unit_v == 2) {
    *focal = focal_mm / (ccd_width * 25.4) * max_size;
    return true;
  }
  return false;
}

bool ReadImageHeader(const std::vector<uint8_t>& bytes, ImageHeader* out, std::string* why) {
  *out = ImageHeader();
  out->format = Sniff(bytes);
  if (out->format == ImageFormat::JPEG) {
    if (!JpegHeader(bytes, out)) {
      *why = "JPEG without a readable frame header";
      return false;
    }
    out->has_focal = ExifFocalLength(bytes.data(), bytes.size(), std::max(out->width, out->height), &out->focal);
    return true;
  }
  if (out->format == ImageFormat::PNG) {
    if (bytes.size() < 33 || std::memcmp(bytes.data() + 12, "IHDR", 4) != 0) {
      *why = "PNG without an IHDR chunk";
      return false;
    }
    const uint8_t* h = bytes.data() + 16;
    out->width = static_cast<int>(Be32(h));
    out->height = static_cast<int>(Be32(h + 4));
    const int depth = h[8], type = h[9], interlace = h[12];
    if (depth != 8 || interlace != 0 || !(type == 0 || type == 2 || type == 3 || type == 4 || type == 6)) {
      *why = "PNG with bit depth " + std::to_string(depth) + ", colour type " + std::to_string(type) + ", interlace " +
             std::to_string(interlace) + " (8-bit non-interlaced grey, grey + alpha, RGB, RGBA and palette are read)";
      return false;
    }
    if (out->width <= 0 || out->height <= 0 || out->width > (1 << 24) || out->height > (1 << 24)) {
      *why = "PNG with an invalid size";
      return false;
    }
    return true;
  }
  *why = "not a JPEG or PNG file";
  return false;
}

bool DecodePng(const std::vector<uint8_t>& bytes, Pixels* out, std::string* why) {
  ImageHeader hdr;
  if (!ReadImageHeader(bytes, &hdr, why)) return false;
  if (hdr.format != ImageFormat::PNG) {
    *why = "not a PNG file";
    return false;
  }
  const int type = bytes[16 + 9];
  const int spp = type == 0 ? 1 : type == 2 ? 3 : type == 3 ? 1 : type == 4 ? 2 : 4;  // samples per pixel
  std::vector<uint8_t> idat, plte;
  size_t i = 8;
  bool end = false;
  while (i + 12 <= bytes.size()) {
    const uint32_t len = Be32(bytes.data() + i);
    if (len > bytes.size() - i - 12) break;
    const uint8_t* type_p = bytes.data() + i + 4;
    const uint32_t crc = Be32(bytes.data() + i + 8 + len);
    if (zlib().crc32(0, type_p, 4 + len) != crc) {
      *why = "PNG chunk with a bad CRC";
      return false;
    }
    if (std::memcmp(type_p, "IDAT", 4) == 0) idat.insert(idat.end(), type_p + 4, type_p + 4 + len);
    if (std::memcmp(type_p, "PLTE", 4) == 0) plte.assign(type_p + 4, type_p + 4 + len);
    if (std::memcmp(type_p, "IEND", 4) == 0) {
      end = true;
      break;
    }
    i += 12 + len;
  }
  if (!end || idat.empty()) {
    *why = "truncated PNG";
    return false;
  }
  if (type == 3 && (plte.empty() || plte.size() % 3 != 0)) {
    *why = "palette PNG without a valid PLTE chunk";
    return false;
  }
  const int W = hdr.width, H = hdr.height;
  const size_t row = static_cast<size_t>(W) * spp;
  // deflate expands at most 1032:1, so a header that claims more than that is corrupt: refuse it before allocating
  if (static_cast<double>(row + 1) * H > 1032.0 * static_cast<double>(idat.size()) + 1024.0) {
    *why = "PNG whose image data is too short for its size";
    return false;
  }
  std::vector<uint8_t> raw((row + 1) * H);
  unsigned long n = raw.size();
  if (zlib().uncompress(raw.data(), &n, idat.data(), idat.size()) != 0 || n != raw.size()) {
    *why = "PNG image data does not inflate to its size";
    return false;
  }
  // undo the per-row filters (bpp = bytes per complete pixel = spp at bit depth 8)
  std::vector<uint8_t> px(row * H);
  for (int y = 0; y < H; ++y) {
    const uint8_t f = raw[y * (row + 1)];
    const uint8_t* s = raw.data() + y * (row + 1) + 1;
    uint8_t* d = px.data() + y * row;
    const uint8_t* up = y ? d - row : nullptr;
    for (size_t x = 0; x < row; ++x) {
      const int a = x >= static_cast<size_t>(spp) ? d[x - spp] : 0, b = up ? up[x] : 0;
      const int c = (up && x >= static_cast<size_t>(spp)) ? up[x - spp] : 0;
      int v;
      switch (f) {
        case 0: v = s[x]; break;
        case 1: v = s[x] + a; break;
        case 2: v = s[x] + b; break;
        case 3: v = s[x] + ((a + b) >> 1); break;
        case 4: {
          const int p = a + b - c, pa = std::abs(p - a), pb = std::abs(p - b), pc = std::abs(p - c);
          v = s[x] + ((pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c));
          break;
        }
        default:
          *why = "PNG row with an unknown filter type " + std::to_string(f);
          return false;
      }
      d[x] = static_cast<uint8_t>(v);
    }
  }
  out->width = W;
  out->height = H;
  if (type == 0 || type == 2 || type == 6) {
    out->channels = spp;
    out->data = std::move(px);
  } else if (type == 4) {  // grey + alpha: the alpha is ignored
    out->channels = 1;
    out->data.resize(static_cast<size_t>(W) * H);
    for (size_t k = 0; k < out->data.size(); ++k) out->data[k] = px[2 * k];
  } else {  // palette -> RGB
    out->channels = 3;
    out->data.resize(static_cast<size_t>(W) * H * 3);
    const size_t entries = plte.size() / 3;
    for (size_t k = 0; k < static_cast<size_t>(W) * H; ++k) {
      if (px[k] >= entries) {
        *why = "palette PNG with an index outside the palette";
        return false;
      }
      std::memcpy(&out->data[3 * k], &plte[3 * px[k]], 3);
    }
  }
  return true;
}

std::vector<uint8_t> EncodePng(const uint8_t* pixels, int width, int height, int channels) {
  if (width <= 0 || height <= 0 || (channels != 1 && channels != 3 && channels != 4))
    throw std::invalid_argument("[image_reader.cc] Check Failed: a PNG is non-empty with 1, 3 or 4 channels");
  const size_t row = static_cast<size_t>(width) * channels;
  std::vector<uint8_t> raw((row + 1) * height);
  for (int y = 0; y < height; ++y) {  // filter type 0 on every row
    raw[(row + 1) * y] = 0;
    std::memcpy(&raw[(row + 1) * y + 1], pixels + row * y, row);
  }
  unsigned long n = zlib().compress_bound(raw.size());
  std::vector<uint8_t> idat(n);
  if (zlib().compress2(idat.data(), &n, raw.data(), raw.size(), 6) != 0)
    throw std::runtime_error("[image_reader.cc] compress2 failed");
  idat.resize(n);
  std::vector<uint8_t> out = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1a, '\n'};
  auto chunk = [&out](const char* type, const uint8_t* body, size_t len) {
    const uint8_t be[4] = {uint8_t(len >> 24), uint8_t(len >> 16), uint8_t(len >> 8), uint8_t(len)};
    out.insert(out.end(), be, be + 4);
    const size_t at = out.size();
    out.insert(out.end(), type, type + 4);
    out.insert(out.end(), body, body + len);
    const uint32_t crc = static_cast<uint32_t>(zlib().crc32(0, &out[at], static_cast<unsigned>(4 + len)));
    const uint8_t bc[4] = {uint8_t(crc >> 24), uint8_t(crc >> 16), uint8_t(crc >> 8), uint8_t(crc)};
    out.insert(out.end(), bc, bc + 4);
  };
  const uint32_t w = static_cast<uint32_t>(width), h = static_cast<uint32_t>(height);
  const uint8_t color_type = channels == 1 ? 0 : (channels == 3 ? 2 : 6);
  const uint8_t ihdr[13] = {uint8_t(w >> 24), uint8_t(w >> 16), uint8_t(w >> 8), uint8_t(w), uint8_t(h >> 24),
                            uint8_t(h >> 16), uint8_t(h >> 8), uint8_t(h), 8, color_type, 0, 0, 0};
  chunk("IHDR", ihdr, 13);
  chunk("IDAT", idat.data(), idat.size());
  chunk("IEND", nullptr, 0);
  return out;
}

std::vector<uint8_t> ToGrey(const Pixels& p) {
  const size_t n = static_cast<size_t>(p.width) * p.height;
  if (p.channels == 1) return p.data;
  std::vector<uint8_t> g(n);
  for (size_t k = 0; k < n; ++k) {
    const uint8_t* s = &p.data[k * p.channels];
    volatile float v = 0.2126f * static_cast<float>(s[0]);  // rounded per operation, in this order
    v = v + 0.7152f * static_cast<float>(s[1]);
    v = v + 0.0722f * static_cast<float>(s[2]);
    g[k] = static_cast<uint8_t>(v + 0.5f);
  }
  return g;
}

std::vector<std::string> ListImages(const std::string& image_path, const std::vector<std::string>& image_list) {
  if (!image_list.empty()) return image_list;
  namespace fs = std::filesystem;
  std::vector<std::string> names;
  const fs::path root(image_path);
  for (const auto& e : fs::recursive_directory_iterator(root)) {
    if (!e.is_regular_file()) continue;
    names.push_back(e.path().lexically_relative(root).generic_string());
  }
  std::sort(names.begin(), names.end());
  return names;
}

ImageReader::ImageReader(const ImageReaderOptions& options, CameraMode mode, const std::string& image_path,
                         const std::vector<std::string>& image_list, Database* db)
    : options_(options), mode_(mode), image_path_(image_path), names_(ListImages(image_path, image_list)), db_(db) {
  model_ = CameraModelId(options_.camera_model);
  if (options_.existing_camera_id != -1) prev_camera_ = db_->ReadCamera(options_.existing_camera_id);
}

void ImageReader::Warn(const std::string& name, const std::string& what) {
  fprintf(stderr, "W [image_reader.cc] %s: %s, skipped\n", name.c_str(), what.c_str());
}

void ImageReader::Load(size_t index, Item* item) const {
  item->name = names_.at(index);
  item->path = (std::filesystem::path(image_path_) / item->name).string();
  item->bytes = ReadFileBytes(item->path);
  item->error.clear();
  if (item->bytes.empty()) item->error = "cannot read the file";
  else ReadImageHeader(item->bytes, &item->header, &item->error);
}

ImageReader::Status ImageReader::Assign(Item* item) {
  const std::string& name = item->name;
  auto warn = [&](const std::string& what) { Warn(name, what); };
  ImageRow existing;
  if (db_->ReadImageWithName(name, &existing)) {
    warn("already in the database");
    return Status::IMAGE_EXISTS;
  }
  if (!item->error.empty()) {
    warn(item->error);
    return Status::BITMAP_ERROR;
  }
  const ImageHeader& h = item->header;
  const size_t slash = name.rfind('/');
  const std::string folder = slash == std::string::npos ? "" : name.substr(0, slash);
  const bool have = prev_camera_.camera_id != 0;
  if (options_.existing_camera_id != -1) {
    if (prev_camera_.width != h.width || prev_camera_.height != h.height) {
      warn("size differs from the existing camera " + std::to_string(options_.existing_camera_id));
      return Status::CAMERA_EXIST_DIM_ERROR;
    }
  } else {
    if (have && (mode_ == CameraMode::SINGLE || (mode_ == CameraMode::PER_FOLDER && folder == prev_folder_)) &&
        (prev_camera_.width != h.width || prev_camera_.height != h.height)) {
      warn("size differs from the shared camera");
      return Status::CAMERA_SINGLE_DIM_ERROR;
    }
    if (!have || mode_ == CameraMode::AUTO || mode_ == CameraMode::PER_IMAGE ||
        (mode_ == CameraMode::PER_FOLDER && folder != prev_folder_)) {
      CameraRow c;
      c.model = model_;
      c.width = h.width;
      c.height = h.height;
      if (options_.camera_params.empty()) {
        double f = h.focal;
        c.has_prior_focal_length = h.has_focal;
        if (!h.has_focal) f = options_.default_focal_length_factor * std::max(h.width, h.height);
        c.params = InitialCameraParams(model_, f, h.width, h.height);
      } else {
        c.params = CsvToDoubles(options_.camera_params);
        c.has_prior_focal_length = true;
      }
      c.camera_id = db_->AddCamera(c.model, c.width, c.height, c.params, c.has_prior_focal_length);
      prev_camera_ = c;
    }
  }
  item->camera = prev_camera_;
  prev_folder_ = folder;
  return Status::SUCCESS;
}

}  // namespace b2mh
