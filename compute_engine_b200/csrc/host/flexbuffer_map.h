// flexbuffer_map.h -- minimal FlexBuffers support for the op attributes.
//
// The reference reads its custom-op attributes with flatbuffers' flexbuffers
// library (LCE/tflite/kernels/bconv2d.cc:89-124, bmaxpool.cc:24-31), which is not
// vendored and cannot be linked here. The attributes are always ONE map of scalars: integers
// written by LCE/mlir/ir/lce_ops.cc:36-64, and ints, floats and bools for
// TFLite_Detection_PostProcess. So a map reader (and, for the
// synthetic-model writer and the tests, a map writer) is all that is needed. The
// wire format is restated from the FlexBuffers format and pinned by the byte blobs
// the reference's own tests hold (LCE/mlir/tests/legalize-lce.mlir:9,21) in
// tests/test_host_ops.py.
#ifndef LCE_B200_HOST_FLEXBUFFER_MAP_H_
#define LCE_B200_HOST_FLEXBUFFER_MAP_H_

#include <cstddef>
#include <cstdint>
#include <string>
#include <utility>
#include <vector>

namespace lce_b200 {

class FlexMap {
 public:
  // Parses `buffer` (borrowed; must outlive the object). ok() is false if the
  // root is not a map or the buffer is malformed; lookups then report "null",
  // like flexbuffers' Reference::IsNull() on a missing key.
  FlexMap(const uint8_t* buffer, size_t length);
  bool ok() const { return ok_; }
  size_t size() const { return keys_.size(); }
  bool Has(const char* key) const;
  // AsInt32() semantics: INT / UINT / BOOL / FLOAT scalars convert; missing -> 0.
  int32_t AsInt32(const char* key) const;
  // A FLOAT (byte width 4 or 8), INT, UINT or BOOL scalar as a float / as a bool (nonzero);
  // default_value for a missing key or a value that is not a number.
  float AsFloat(const char* key, float default_value) const;
  bool AsBool(const char* key, bool default_value) const;
  const std::vector<std::string>& keys() const { return keys_; }

 private:
  int Find(const char* key) const;
  bool IsNumber(int i) const;
  bool ok_ = false;
  std::vector<std::string> keys_;
  std::vector<int64_t> values_;
  std::vector<double> reals_;
  std::vector<int> types_;   // FlexBuffers type of each value
};

// Serialises {key: int} pairs the way flexbuffers::Builder does for small maps
// (keys sorted by strcmp, one shared byte width).
std::vector<uint8_t> WriteFlexIntMap(std::vector<std::pair<std::string, int64_t>> items);

}  // namespace lce_b200
#endif
