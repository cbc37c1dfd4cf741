// image_reader.h -- the host half of feature extraction from image files: what COLMAP's ImageReader
// (U:controllers/image_reader.cc, COLMAP 3.9.1) and Bitmap (U:sensor/bitmap.cc) do before the pixels reach SIFT, and
// the pycolmap functions above them (R:pycolmap/pipeline/images.h:24-94, R:pycolmap/pipeline/extract_features.h:23-61).
// SURVEY.md rows U1-U6.
//   file list      the sorted recursive walk of image_path, or image_list; names relative, '/'-separated
//   format         from the magic bytes: JPEG goes whole to the device (nvJPEG), PNG is decoded here (zlib bound at
//                  run time from libz.so.1), anything else is skipped with a warning
//   header / EXIF  JPEG SOF / PNG IHDR give the size; Bitmap::ExifFocalLength's rules give the focal length
//   cameras        ImageReader::Next's camera assignment per CameraMode / existing_camera_id
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "database.h"

namespace b2mh {

enum class CameraMode { AUTO = 0, SINGLE = 1, PER_FOLDER = 2, PER_IMAGE = 3 };  // R:pycolmap/pipeline/images.h:151-156

// ImageReaderOptions as pycolmap binds it (R:pycolmap/pipeline/images.h:158-201; defaults U:controllers/image_reader.h)
struct ImageReaderOptions {
  std::string camera_model = "SIMPLE_RADIAL";
  std::string mask_path;
  int existing_camera_id = -1;
  std::string camera_params;
  double default_focal_length_factor = 1.2;
  std::string camera_mask_path;
};

// camera model name -> COLMAP model id, -1 when unknown (ExistsCameraModelWithName)
int CameraModelId(const std::string& name);
// VerifyCameraParams: empty params are valid; otherwise the comma-separated list has the model's parameter count
bool VerifyCameraParams(const std::string& model, const std::string& params);
// CameraModel::InitializeParams: focal lengths f, principal point (w / 2, h / 2), the rest 0 (FOV's omega 1e-2)
std::vector<double> InitialCameraParams(int model, double focal, int64_t width, int64_t height);

enum class ImageFormat { UNKNOWN = 0, JPEG, PNG };

// What the header says: format, size, the EXIF focal length (Bitmap::ExifFocalLength) when there is one.
struct ImageHeader {
  ImageFormat format = ImageFormat::UNKNOWN;
  int width = 0, height = 0;
  bool has_focal = false;
  double focal = 0.0;
};

std::vector<uint8_t> ReadFileBytes(const std::string& path);  // empty when unreadable
// false (with *why) for a format or a PNG variant this reader does not take, or a truncated header
bool ReadImageHeader(const std::vector<uint8_t>& bytes, ImageHeader* out, std::string* why);
// Bitmap::ExifFocalLength on the EXIF block of a JPEG (APP1); max_size = max(width, height) of the image
bool ExifFocalLength(const uint8_t* data, size_t size, double max_size, double* focal);

// A decoded PNG: 8-bit samples, channels 1 (grey, and grey + alpha with the alpha dropped), 3 (RGB, palette expanded)
// or 4 (RGBA).  False (with *why) for 16-bit, interlaced, other bit depths, a bad CRC or a corrupt stream.
struct Pixels {
  int width = 0, height = 0, channels = 0;
  std::vector<uint8_t> data;  // packed rows
};
bool DecodePng(const std::vector<uint8_t>& bytes, Pixels* out, std::string* why);
// An 8-bit PNG of packed rows (1 grey, 3 RGB or 4 RGBA channels), compressed with zlib's compress2 (level 6), every
// row with filter type 0.
std::vector<uint8_t> EncodePng(const uint8_t* pixels, int width, int height, int channels);
// FreeImage's ConvertToGreyscale on host pixels (the same Rec709 rule as the device kernel); 1 channel passes through
std::vector<uint8_t> ToGrey(const Pixels& p);

// The file list of ImageReaderOptions: names (relative to image_path, '/'-separated) in reading order.
std::vector<std::string> ListImages(const std::string& image_path, const std::vector<std::string>& image_list);

// ImageReader::Next's per-image decisions, in two halves: Load() reads file `index` and its header and touches no
// database (so that a reader thread can run it ahead); Assign() takes the loaded images in order, assigns each a camera
// (writing a new one to `db`) and returns SUCCESS, or the reason the image is skipped.  A warning is printed for every
// skip.
class ImageReader {
 public:
  enum class Status { SUCCESS, IMAGE_EXISTS, BITMAP_ERROR, CAMERA_SINGLE_DIM_ERROR, CAMERA_EXIST_DIM_ERROR };
  struct Item {
    std::string name, path;
    std::vector<uint8_t> bytes;
    ImageHeader header;
    std::string error;  // why the file or its header could not be read
    CameraRow camera;
  };
  ImageReader(const ImageReaderOptions& options, CameraMode mode, const std::string& image_path,
              const std::vector<std::string>& image_list, Database* db);
  size_t NumImages() const { return names_.size(); }
  void Load(size_t index, Item* item) const;
  Status Assign(Item* item);
  static void Warn(const std::string& name, const std::string& what);

 private:
  ImageReaderOptions options_;
  CameraMode mode_;
  std::string image_path_;
  std::vector<std::string> names_;
  Database* db_;
  int model_ = -1;
  CameraRow prev_camera_;  // camera_id 0 = none yet
  std::string prev_folder_;
};

}  // namespace b2mh
