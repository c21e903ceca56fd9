// Frame resampling of the System-1 input preprocessing (SURVEY.md §8 row a12): the reference resizes every RGB / depth
// frame with Pillow's `Image.resize((224, 224))` (internnav/agent/internvla_n1_agent.py L309-321) -- a two-pass
// separable bicubic (a = -0.5) with antialiasing, 22-bit fixed-point weights for 8-bit images and double accumulation
// for float images (Pillow src/libImaging/Resample.c, restated in oracle/pil_resize.py and pinned there bit for bit).
// The kernels below reproduce it bit-exactly for a batch of frames resident in HBM.
#pragma once
#include <vector>

#include "n1_ops.h"

namespace n1 {

struct ResizeCoeffs {
  int in_size = 0, out_size = 0, ksize = 0;
  std::vector<int32_t> bounds;   // [out, 2] = (first input index, window length)
  std::vector<double> weights;   // [out, ksize] normalised, zero-padded
  std::vector<int32_t> fixed;    // [out, ksize] round-half-away(weights * 2^22)
};
// precompute_coeffs + normalize_coeffs_8bpc (host)
void resize_coeffs(int in_size, int out_size, ResizeCoeffs& c);

struct ResizePlan {
  int in_h = 0, in_w = 0, out_h = 0, out_w = 0;
  ResizeCoeffs h, v;             // horizontal (width) and vertical (height) tables, host copies
  int32_t *h_bounds = nullptr, *v_bounds = nullptr, *h_fixed = nullptr, *v_fixed = nullptr;
  double *h_w = nullptr, *v_w = nullptr;
  ResizePlan(int in_h, int in_w, int out_h, int out_w, cudaStream_t s);
  ~ResizePlan();
  size_t workspace_bytes(int n, int channels, bool is_float) const;
};

// src uint8 [n, in_h, in_w, 3] -> dst_f32 [n, out_h, out_w, 3] = resized / 255 (fp32 division) and / or dst_u8 (either
// may be null).  ws: workspace_bytes(n, 3, false).
void resize_rgb_u8(const ResizePlan& p, const uint8_t* src, int n, float* dst_f32, uint8_t* dst_u8, void* ws,
                   cudaStream_t s);
// src float [n, in_h, in_w] -> dst float [n, out_h, out_w] = min(resized * mul, clip_max)  (fp32 multiply; pass
// clip_max = +inf for none).  ws: workspace_bytes(n, 1, true).
void resize_f32(const ResizePlan& p, const float* src, int n, float mul, float clip_max, float* dst, void* ws,
                cudaStream_t s);

// System-2 image rows (vl_patch.cu).  The Qwen2-VL image processor resizes each image with Pillow to a multiple of 28
// and then rescales, normalises and patchifies it; after a uint8 resize, rescale + normalise is a per-channel table of
// the 256 byte values, so the rows are table lookups of the resized frame's bytes.
struct VlImage {       // layout of n1_vl_image
  const uint8_t* src;  // resized frame [h, w, 3], device
  int32_t h, w;        // multiples of 28
  int64_t row0;        // first output row = rows of the images before it
};
size_t vl_patchify_workspace_bytes(int n_img);
// images HOST [n_img]; lut bf16 [3, 256]; out bf16 [n_rows, 1176] (16-byte aligned), n_rows = sum h * w / 196;
// ws: vl_patchify_workspace_bytes(n_img) (receives the table)
void vl_patchify(const VlImage* images, int n_img, const bf16* lut, bf16* out, long n_rows, void* ws, cudaStream_t s);

}  // namespace n1
