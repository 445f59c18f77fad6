// The device steps nb_eval_image and nb_vis_frame share: the ray of each set pixel of mask_at_box (the mask's exclusive
// prefix count, a CUB scan) and cv2.imwrite's conversion of a float64 image to uint8.
#pragma once
#include <climits>

#include <cub/device/device_scan.cuh>
#include <thrust/iterator/transform_iterator.h>

namespace nb {
namespace {

struct NonZero {
    __host__ __device__ int operator()(unsigned char m) const { return m != 0; }
};

inline cudaError_t scan_mask(void* scratch, size_t& bytes, const unsigned char* mask, int* offset, int n, cudaStream_t s) {
    return cub::DeviceScan::ExclusiveSum(scratch, bytes, thrust::make_transform_iterator(mask, NonZero{}), offset, n, s);
}

// scan_mask's scratch bytes for n pixels; 0 when the size query fails
inline size_t scan_bytes(int n) {
    size_t b = 0;
    if (scan_mask(nullptr, b, nullptr, nullptr, n, 0) != cudaSuccess) { cudaGetLastError(); return 0; }
    return b;
}

// saturate_cast<uchar>(v * 255): cvRound (nearest-even; NaN or outside int32 -> INT_MIN), then clamped to [0, 255]
__device__ __forceinline__ unsigned char to_u8(double v) {
    const double r = rint(__dmul_rn(v, 255.0));
    const int i = (r >= -2147483648.0 && r <= 2147483647.0) ? (int)r : INT_MIN;
    return (unsigned char)min(max(i, 0), 255);
}

}  // namespace
}  // namespace nb
