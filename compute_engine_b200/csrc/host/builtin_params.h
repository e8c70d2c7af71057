// builtin_params.h -- parameter blob handed to this host's builtin registrations as
// node->builtin_data (filled by tflite_model.cc from the flatbuffer's builtin option
// tables, schema.fbs:806-1106). Private to this host: TFLite's own builtin_op_data.h
// structs are not part of the custom-op ABI.
#ifndef LCE_B200_HOST_BUILTIN_PARAMS_H_
#define LCE_B200_HOST_BUILTIN_PARAMS_H_
#include <cstdint>

#include "lce_b200_tflite.h"

namespace lce_b200 {
struct BuiltinParams {
  int32_t builtin_code;
  int32_t padding, stride_h, stride_w, dilation_h, dilation_w;
  int32_t filter_h, filter_w, depth_multiplier;
  int32_t activation;
  int32_t keep_dims;
  int32_t axis;
  float beta;
  int32_t n_new_shape;
  int32_t new_shape[8];
  // STRIDED_SLICE (StridedSliceOptions) and SPLIT (SplitOptions)
  int32_t begin_mask, end_mask, ellipsis_mask, new_axis_mask, shrink_axis_mask, offset;
  int32_t num_splits;
  // RESIZE_BILINEAR (ResizeBilinearOptions) and RESIZE_NEAREST_NEIGHBOR (ResizeNearestNeighborOptions)
  int32_t align_corners, half_pixel_centers;
  // ARG_MAX (ArgMaxOptions): the output's TensorType code
  int32_t output_type;
  // DEPTH_TO_SPACE (DepthToSpaceOptions)
  int32_t block_size;
};

// builtin_data of the "LceBfc[+MUL+ADD]+REDUCE_MAX[+LceQuantize]" node Graph::FuseBinaryFcMax creates
// (builtin_ops.cc runs it): the FULLY_CONNECTED's, the ADD's (zeros without it) and the REDUCE_MAX's
// parameters, K, the points per image, and whether the node stores the float max and its signs.
struct BinaryFcMaxParams {
  BuiltinParams fc, add, reduce;
  int32_t channels_in, points, store_max, store_signs;
};

// ARG_MAX's axis: a constant int32 or int64 tensor of one element (0-D or [1]) in host memory, within
// [-rank, rank) and normalised to [0, rank). Returns nullptr, or why the axis is refused.
// builtin_ops.cc; Graph::FuseResizeArgmax reads the axis through it too.
const char* ArgMaxAxis(const TfLiteTensor* axis, int rank, int* out);

// STRIDED_SLICE's bounds for an input of dims[0..rank) and n = the length of begin / end / strides,
// normalised as TFLite's strided_slice.cc does (masks, negative indices, clamping): the output is
// dims with axis k cut to [begin[k], end[k]). Only the form x[..., a:b] lowers to is taken: unit
// strides and at most one axis not whole. Returns nullptr, or why the slice is refused.
// builtin_ops.cc; Graph::FuseDenseBlocks matches slices through it too.
struct SliceBounds {
  int rank;
  int begin[4], end[4];
};
const char* StridedSliceBounds(const int32_t* dims, int rank, const int32_t* begin, const int32_t* end,
                               const int32_t* strides, int n, const BuiltinParams& p, SliceBounds* out);
}  // namespace lce_b200
#endif
