// System-2 image rows from resized uint8 frames: the rescale, normalise and patchify of the Qwen2-VL image processor
// (Qwen2VLImageProcessorPil._preprocess) for every image of a call in one launch.  See resize.h.
#include "resize.h"

namespace n1 {

namespace {

constexpr int kPatch = 14;                           // patch_size
constexpr int kRowElems = 3 * 2 * kPatch * kPatch;   // channel x temporal_patch_size x 14 x 14 = 1176
constexpr int kChunk = 8;                            // bf16 per 16-byte store
constexpr int kChunks = kRowElems / kChunk;          // 147 stores per row

// blockIdx.y = image, one thread per 16-byte chunk of its rows; consecutive threads write consecutive chunks of a row.
// Row r of an image is sub-patch (r % 4) / 2, (r % 4) % 2 of merged block r / 4 (row-major over gh / 2 x gw / 2);
// element e = c * 392 + t * 196 + py * 14 + px reads pixel (py, px) of that patch, channel c, for both t.
__global__ void __launch_bounds__(256) vl_patchify_kernel(const VlImage* __restrict__ images,
                                                          const uint16_t* __restrict__ lut, uint4* __restrict__ out) {
  const VlImage im = images[blockIdx.y];
  const int gw = im.w / kPatch;
  const long q = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= (long)(im.h / kPatch) * gw * kChunks) return;
  const int r = (int)(q / kChunks), k = (int)(q % kChunks);
  const int b = r >> 2, sub = r & 3, mw = gw >> 1;
  const int y0 = ((b / mw) * 2 + (sub >> 1)) * kPatch, x0 = ((b % mw) * 2 + (sub & 1)) * kPatch;
  const uint8_t* src = im.src + ((long)y0 * im.w + x0) * 3;
  uint32_t v[kChunk / 2];
#pragma unroll
  for (int j = 0; j < kChunk; ++j) {
    const int e = k * kChunk + j, c = e / (2 * kPatch * kPatch), s = e % (kPatch * kPatch);
    const uint32_t x = __ldg(lut + c * 256 + __ldg(src + ((s / kPatch) * im.w + s % kPatch) * 3 + c));
    v[j >> 1] = (j & 1) ? (v[j >> 1] | (x << 16)) : x;
  }
  out[(im.row0 + r) * kChunks + k] = make_uint4(v[0], v[1], v[2], v[3]);
}

}  // namespace

size_t vl_patchify_workspace_bytes(int n_img) { return ((size_t)(n_img > 0 ? n_img : 0) * sizeof(VlImage) + 255) & ~size_t(255); }

void vl_patchify(const VlImage* images, int n_img, const bf16* lut, bf16* out, long n_rows, void* ws, cudaStream_t s) {
  N1_CHECK(n_img > 0 && n_img <= 65535, "vl_patchify: 1..65535 images");
  N1_CHECK(images && lut && out && ws, "vl_patchify: null arguments");
  N1_CHECK(reinterpret_cast<uintptr_t>(out) % 16 == 0, "vl_patchify: output must be 16-byte aligned");
  long rows = 0, max_rows = 0;
  for (int i = 0; i < n_img; ++i) {
    const VlImage& im = images[i];
    N1_CHECK(im.src, "vl_patchify: null frame " + std::to_string(i));
    N1_CHECK(im.h > 0 && im.w > 0 && im.h % (2 * kPatch) == 0 && im.w % (2 * kPatch) == 0,
             "vl_patchify: frame " + std::to_string(i) + " is " + std::to_string(im.h) + " x " + std::to_string(im.w) +
                 "; both sizes must be positive multiples of 28");
    N1_CHECK(im.row0 == rows, "vl_patchify: frame " + std::to_string(i) + " starts at row " + std::to_string(im.row0) +
                                  ", expected " + std::to_string(rows));
    const long n = (long)(im.h / kPatch) * (im.w / kPatch);
    rows += n;
    if (n > max_rows) max_rows = n;
  }
  N1_CHECK(rows == n_rows, "vl_patchify: the frames make " + std::to_string(rows) + " rows, not " + std::to_string(n_rows));
  N1_CUDA(cudaMemcpyAsync(ws, images, (size_t)n_img * sizeof(VlImage), cudaMemcpyHostToDevice, s));
  const dim3 grid((unsigned)((max_rows * kChunks + 255) / 256), (unsigned)n_img);
  vl_patchify_kernel<<<grid, 256, 0, s>>>(static_cast<const VlImage*>(ws), reinterpret_cast<const uint16_t*>(lut),
                                          reinterpret_cast<uint4*>(out));
  prof_count_launch();
  N1_CUDA(cudaGetLastError());
}

}  // namespace n1
