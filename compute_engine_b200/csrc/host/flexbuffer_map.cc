#include "flexbuffer_map.h"

#include <algorithm>
#include <cstring>

namespace lce_b200 {
namespace {

enum FlexType { kNull = 0, kInt = 1, kUInt = 2, kFloat = 3, kKey = 4, kString = 5,
                kIndirectInt = 6, kIndirectUInt = 7, kIndirectFloat = 8, kMap = 9,
                kVector = 10, kBool = 26 };

struct Cursor {
  const uint8_t* base;
  size_t len;
  bool in(size_t off, size_t n) const { return off <= len && n <= len - off; }
  bool ReadU(size_t off, int width, uint64_t* v) const {
    if (!in(off, width)) return false;
    uint64_t r = 0;
    memcpy(&r, base + off, width);  // little endian
    *v = r;
    return true;
  }
  bool ReadI(size_t off, int width, int64_t* v) const {
    uint64_t u;
    if (!ReadU(off, width, &u)) return false;
    const int shift = 64 - 8 * width;
    *v = static_cast<int64_t>(u << shift) >> shift;
    return true;
  }
};

// *out is the scalar as AsInt32 converts it, *real the same scalar as a double.
bool ReadScalar(const Cursor& c, size_t slot, int slot_width, uint8_t packed, int64_t* out, double* real) {
  const int type = packed >> 2;
  const int child_width = 1 << (packed & 3);
  *real = 0.0;
  switch (type) {
    case kInt:
      if (!c.ReadI(slot, slot_width, out)) return false;
      *real = static_cast<double>(*out);
      return true;
    case kUInt:
    case kBool: {
      uint64_t u;
      if (!c.ReadU(slot, slot_width, &u)) return false;
      *out = static_cast<int64_t>(u);
      *real = static_cast<double>(u);
      return true;
    }
    case kFloat: {
      if (slot_width == 4) {
        float f;
        if (!c.in(slot, 4)) return false;
        memcpy(&f, c.base + slot, 4);
        *out = static_cast<int64_t>(f);
        *real = f;
        return true;
      }
      if (slot_width == 8) {
        double d;
        if (!c.in(slot, 8)) return false;
        memcpy(&d, c.base + slot, 8);
        *out = static_cast<int64_t>(d);
        *real = d;
        return true;
      }
      return false;
    }
    case kIndirectInt:
    case kIndirectUInt: {
      uint64_t off;
      if (!c.ReadU(slot, slot_width, &off) || off > slot) return false;
      if (type == kIndirectInt) return c.ReadI(slot - off, child_width, out);
      uint64_t u;
      if (!c.ReadU(slot - off, child_width, &u)) return false;
      *out = static_cast<int64_t>(u);
      return true;
    }
    default:
      *out = 0;  // non-scalar: AsInt32() of a map/vector/string is not used here
      return true;
  }
}

}  // namespace

FlexMap::FlexMap(const uint8_t* buffer, size_t length) {
  if (!buffer || length < 3) return;
  Cursor c{buffer, length};
  const int root_width = buffer[length - 1];
  const uint8_t root_packed = buffer[length - 2];
  if (root_width != 1 && root_width != 2 && root_width != 4 && root_width != 8) return;
  if ((root_packed >> 2) != kMap) return;
  if (length < static_cast<size_t>(root_width) + 2) return;
  const size_t root_slot = length - 2 - root_width;
  uint64_t off;
  if (!c.ReadU(root_slot, root_width, &off) || off > root_slot) return;
  const size_t map = root_slot - off;  // address of the first value
  const int w = 1 << (root_packed & 3);
  if (map < static_cast<size_t>(3 * w)) return;
  uint64_t n, keys_width, keys_off;
  if (!c.ReadU(map - w, w, &n) || !c.ReadU(map - 2 * w, w, &keys_width) ||
      !c.ReadU(map - 3 * w, w, &keys_off))
    return;
  if (n > 4096 || keys_off > map - 3 * w) return;
  if (keys_width != 1 && keys_width != 2 && keys_width != 4 && keys_width != 8) return;
  const size_t keys = map - 3 * w - keys_off;
  const size_t types = map + n * w;
  if (!c.in(types, n)) return;
  for (uint64_t i = 0; i < n; ++i) {
    const size_t kslot = keys + i * keys_width;
    uint64_t koff;
    if (!c.ReadU(kslot, static_cast<int>(keys_width), &koff) || koff > kslot) return;
    const size_t kaddr = kslot - koff;
    const void* nul = memchr(buffer + kaddr, 0, length - kaddr);
    if (!nul) return;
    keys_.emplace_back(reinterpret_cast<const char*>(buffer + kaddr));
    int64_t v;
    double real;
    if (!ReadScalar(c, map + i * w, w, buffer[types + i], &v, &real)) return;
    values_.push_back(v);
    reals_.push_back(real);
    types_.push_back(buffer[types + i] >> 2);
  }
  ok_ = true;
}

bool FlexMap::Has(const char* key) const {
  if (!ok_) return false;
  return std::find(keys_.begin(), keys_.end(), key) != keys_.end();
}

int32_t FlexMap::AsInt32(const char* key) const {
  if (!ok_) return 0;
  for (size_t i = 0; i < keys_.size(); ++i)
    if (keys_[i] == key) return static_cast<int32_t>(values_[i]);
  return 0;
}

int FlexMap::Find(const char* key) const {
  if (!ok_) return -1;
  for (size_t i = 0; i < keys_.size(); ++i)
    if (keys_[i] == key) return static_cast<int>(i);
  return -1;
}

bool FlexMap::IsNumber(int i) const {
  return i >= 0 && (types_[i] == kInt || types_[i] == kUInt || types_[i] == kFloat || types_[i] == kBool ||
                    types_[i] == kIndirectInt || types_[i] == kIndirectUInt);
}

float FlexMap::AsFloat(const char* key, float default_value) const {
  const int i = Find(key);
  if (!IsNumber(i)) return default_value;
  return (types_[i] == kIndirectInt || types_[i] == kIndirectUInt) ? static_cast<float>(values_[i])
                                                                   : static_cast<float>(reals_[i]);
}

bool FlexMap::AsBool(const char* key, bool default_value) const {
  const int i = Find(key);
  if (!IsNumber(i)) return default_value;
  return types_[i] == kFloat ? reals_[i] != 0.0 : values_[i] != 0;
}

std::vector<uint8_t> WriteFlexIntMap(std::vector<std::pair<std::string, int64_t>> items) {
  // Key strings are emitted in insertion order (as flexbuffers::Builder does when
  // the caller adds keys one by one); the keys vector and the values are sorted.
  std::vector<size_t> order(items.size());
  for (size_t i = 0; i < order.size(); ++i) order[i] = i;
  std::sort(order.begin(), order.end(), [&](size_t a, size_t b) {
    return strcmp(items[a].first.c_str(), items[b].first.c_str()) < 0;
  });
  for (int log2w = 0; log2w < 3; ++log2w) {
    const int w = 1 << log2w;
    const int64_t lim = (int64_t{1} << (8 * w - 1));
    std::vector<uint8_t> out;
    std::vector<size_t> key_pos(items.size());
    for (size_t i = 0; i < items.size(); ++i) {
      key_pos[i] = out.size();
      out.insert(out.end(), items[i].first.begin(), items[i].first.end());
      out.push_back(0);
    }
    auto align = [&]() { while (out.size() % w) out.push_back(0); };
    auto put = [&](uint64_t v) { for (int b = 0; b < w; ++b) out.push_back((v >> (8 * b)) & 0xFF); };
    bool fits = true;
    align();
    put(items.size());                       // keys vector: size, then offsets
    const size_t keys_vec = out.size();
    for (size_t i : order) {
      const uint64_t off = out.size() - key_pos[i];
      if (off >= (uint64_t{1} << (8 * w))) fits = false;
      put(off);
    }
    align();
    put(out.size() - keys_vec);              // map prefix: keys offset, keys width, size
    put(w);
    put(items.size());
    const size_t map = out.size();
    for (size_t i : order) {
      if (items[i].second >= lim || items[i].second < -lim) fits = false;
      put(static_cast<uint64_t>(items[i].second));
    }
    for (size_t i = 0; i < items.size(); ++i) out.push_back((kInt << 2) | log2w);
    align();
    if (out.size() - map >= (uint64_t{1} << (8 * w))) fits = false;
    if (!fits) continue;
    put(out.size() - map);
    out.push_back((kMap << 2) | log2w);
    out.push_back(static_cast<uint8_t>(w));
    return out;
  }
  return {};
}

}  // namespace lce_b200
