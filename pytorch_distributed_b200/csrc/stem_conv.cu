// ResNet stem convolution (7x7, stride 2, pad 3, C_in = 3) as im2col + the wgmma GEMM of gemm_bnstats.cu (sm_90a).
//
// cuDNN serves this layer with legacy kernels (C_in = 3 fits no tensor-core tile; padding C_in to 4 or 8 does not help,
// tools/conv_stem_probe.py).  The layer is only 60 GFLOP; written as a GEMM it is bound by its 411 MB output:
//   A[M, 192]  = im2col(x)        M = N*OH*OW output pixels, one 384-byte row per pixel        (this file)
//   Y[M, 64]   = A x Wp^T         persistent wgmma GEMM, BatchNorm statistics in its epilogue    (gemm_bnstats.cu)
//   dWp[64,192]= dY^T x A         library GEMM over the saved A                                  (ops/stem_conv.py)
// K ordering of a row: k = r*24 + s*3 + c for filter row r < 7, filter column s < 7, channel c < 3; positions with
// s*3 + c >= 21 and k >= 168 are zero (the packed weights are zero there too).  A filter row is 21 CONTIGUOUS input
// elements in NHWC, so a 16-byte granule of A is 8 consecutive input elements: one thread builds one granule.
// im2col only moves 16-bit values, so one pair of kernels serves bf16 and fp16 (A has the input's dtype).
// Reference call site: torchvision resnet.conv1 reached through /root/reference/distributed.py:136-139.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include "common.cuh"
#include "host.h"

namespace ptd {

constexpr int kStemK = 192;            // padded GEMM K (3 x 64)
constexpr int kStemRowK = 24;          // padded elements per filter row (21 real)
constexpr int kStemGranules = kStemK / 8;

// One granule (8 consecutive K positions of one output pixel) the slow way: 8 predicated 2-byte loads.  Used for the
// pixels whose filter window touches the left / right image border and for images with an odd row length.
__device__ __forceinline__ V4 stem_granule_scalar(const unsigned short* __restrict__ row, int e0, int q, int row_elems) {
  unsigned short v[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int sc = q * 8 + j, e = e0 + j;
    v[j] = (sc < 21 && e >= 0 && e < row_elems) ? __ldg(row + e) : (unsigned short)0;
  }
  return V4{(uint32_t)v[0] | ((uint32_t)v[1] << 16), (uint32_t)v[2] | ((uint32_t)v[3] << 16), (uint32_t)v[4] | ((uint32_t)v[5] << 16),
            (uint32_t)v[6] | ((uint32_t)v[7] << 16)};
}

// Fallback (odd row lengths / unaligned base): one granule per thread straight from global memory.
__global__ void __launch_bounds__(256) stem_im2col_scalar_kernel(const unsigned short* __restrict__ x, unsigned short* __restrict__ a, int H,
                                                                 int W, int OH, int OW) {
  const int g = blockIdx.y * blockDim.x + threadIdx.x;       // granule inside the output row
  if (g >= OW * kStemGranules) return;
  const int orow = blockIdx.x;                               // n * OH + oh
  const int n = orow / OH, oh = orow - n * OH;
  const int ow = g / kStemGranules, gq = g - ow * kStemGranules;
  const int r = gq / 3, q = gq - 3 * r;
  const int row_elems = W * 3;
  V4 o{0u, 0u, 0u, 0u};
  const int ih = 2 * oh - 3 + r;
  if (r < 7 && ih >= 0 && ih < H) {
    const unsigned short* row = x + ((int64_t)n * H + ih) * row_elems;
    o = stem_granule_scalar(row, (2 * ow - 3) * 3 + q * 8, q, row_elems);
  }
  st_v4(a + ((int64_t)orow * OW * kStemGranules + g) * 8, o);
}

// One CTA per output row (n, oh).  The seven input rows the row's filter windows touch are staged in shared memory with
// coalesced 16-byte loads (gathering 2-byte elements from global memory costs ~200 instructions per granule), each behind 16 zero elements and followed by 16 more, so the left / right image padding
// and the rows above / below the image are plain zeros in shared memory and EVERY granule takes the same path:
// a filter row's 21 elements start at element (2*ow-3)*3 of the input row - an odd element index, i.e. 2 bytes past a
// 4-byte word - so a granule is five aligned 32-bit shared loads and four PRMTs (hi half of word k | lo half of word k+1).
constexpr int kStemPad = 16;          // zero elements before / after each staged row (multiple of 8: keeps 16-byte alignment)

__global__ void __launch_bounds__(256) stem_im2col_kernel(const unsigned short* __restrict__ x, unsigned short* __restrict__ a, int H, int W,
                                                          int OH, int OW) {
  extern __shared__ __align__(16) unsigned char stem_smem[];
  const int row_elems = W * 3;                               // host guarantees row_elems % 8 == 0 (16-byte rows)
  const int srow = row_elems + 2 * kStemPad;                 // staged row length in elements
  unsigned short* sm = reinterpret_cast<unsigned short*>(stem_smem);
  const int orow = blockIdx.x;                               // n * OH + oh
  const int n = orow / OH, oh = orow - n * OH;
  const int vec_per_row = srow / 8;
  for (int v = threadIdx.x; v < 7 * vec_per_row; v += blockDim.x) {
    const int r = v / vec_per_row, c = v - r * vec_per_row;  // 16-byte vector c of staged row r
    const int ih = 2 * oh - 3 + r;
    const int e = c * 8 - kStemPad;                          // first input element of this vector
    V4 val{0u, 0u, 0u, 0u};
    if (ih >= 0 && ih < H && e >= 0 && e < row_elems)
      val = ld_stream(x + ((int64_t)n * H + ih) * row_elems + e);
    *reinterpret_cast<V4*>(sm + r * srow + c * 8) = val;
  }
  __syncthreads();
  const int total = OW * kStemGranules;
  unsigned short* out = a + (int64_t)orow * total * 8;
  for (int g = threadIdx.x; g < total; g += blockDim.x) {
    const int ow = g / kStemGranules, gq = g - ow * kStemGranules;
    const int r = gq / 3, q = gq - 3 * r;                    // filter row, granule inside the row (r == 7: zero padding of K)
    V4 o{0u, 0u, 0u, 0u};
    if (r < 7) {
      const int e0 = (2 * ow - 3) * 3 + q * 8 + kStemPad;    // odd; >= 7, and e0 + 9 <= srow for every ow
      const uint32_t* w = reinterpret_cast<const uint32_t*>(sm + r * srow + (e0 - 1));
      const uint32_t w0 = w[0], w1 = w[1], w2 = w[2], w3 = w[3], w4 = w[4];
      o.x = __byte_perm(w0, w1, 0x5432);
      o.y = __byte_perm(w1, w2, 0x5432);
      o.z = __byte_perm(w2, w3, 0x5432);
      o.w = __byte_perm(w3, w4, 0x5432);
      if (q == 2) {                                          // positions 21..23 of the filter row are K padding
        o.z &= 0x0000FFFFu;
        o.w = 0u;
      }
    }
    st_v4(out + (int64_t)g * 8, o);
  }
}

// x: [N, 3, H, W] channels_last bf16 or fp16 (physically N x H x W x 3).  returns A (x's dtype) as a [N, 192, OH, OW]
// channels_last view (physically [N*OH*OW, 192] row-major), which is exactly the activation layout conv1x1_bnstats() takes.
at::Tensor stem_im2col(const at::Tensor& x) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 4 && x.size(1) == 3 && (x.scalar_type() == at::kBFloat16 || x.scalar_type() == at::kHalf) &&
                  x.is_contiguous(at::MemoryFormat::ChannelsLast),
              "stem_im2col: x must be a [N, 3, H, W] channels_last bf16 or fp16 CUDA tensor");
  const int64_t N = x.size(0);
  const int H = (int)x.size(2), W = (int)x.size(3);
  const int OH = (H + 6 - 7) / 2 + 1, OW = (W + 6 - 7) / 2 + 1;
  TORCH_CHECK(H >= 7 && W >= 7 && (int64_t)W * 3 < (1 << 30), "stem_im2col: unsupported image size");
  c10::cuda::CUDAGuard guard(x.device());
  at::Tensor a = at::empty({N, OH, OW, kStemK}, x.options());
  TORCH_CHECK(N * OH < ((int64_t)1 << 31) && (int64_t)OW * kStemGranules < (1 << 24), "stem_im2col: too many output rows");
  const unsigned short* xp = reinterpret_cast<const unsigned short*>(x.data_ptr());
  unsigned short* ap = reinterpret_cast<unsigned short*>(a.data_ptr());
  cudaStream_t st = at::cuda::getCurrentCUDAStream();
  const int64_t row_elems = (int64_t)W * 3;
  const size_t smem = (size_t)7 * (row_elems + 2 * kStemPad) * 2;
  // staged path: 16-byte rows (W % 8 == 0: every ImageNet-style size), aligned base, rows that fit the shared memory budget
  if (row_elems % 8 == 0 && (reinterpret_cast<uintptr_t>(x.data_ptr()) & 15) == 0 && smem <= 96 * 1024) {
    if (smem > 48 * 1024) {
      static bool attr_set[64] = {};
      const int dev = x.get_device();
      if (dev >= 0 && dev < 64 && !attr_set[dev]) {
        C10_CUDA_CHECK(cudaFuncSetAttribute(stem_im2col_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
        attr_set[dev] = true;
      }
    }
    stem_im2col_kernel<<<(unsigned)(N * OH), 256, smem, st>>>(xp, ap, H, W, OH, OW);
  } else {
    dim3 grid((unsigned)(N * OH), (unsigned)((OW * kStemGranules + 255) / 256));
    stem_im2col_scalar_kernel<<<grid, 256, 0, st>>>(xp, ap, H, W, OH, OW);
  }
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  return a.permute({0, 3, 1, 2});
}

}  // namespace ptd
