// Host-side declarations shared by the .cu / .cpp translation units and the bindings.
#pragma once
#include <cuda_runtime_api.h>
#include <torch/extension.h>

#include <cstdint>
#include <string>
#include <vector>

#include "comm_types.h"

namespace ptd {

// One contiguous piece of one tensor inside one CTA's arena range (static per plan).
struct Seg {
  int32_t tensor;     // index into the launch's pointer pack
  int32_t len;        // elements
  int64_t src_off;    // element offset inside the tensor
  int64_t arena_off;  // element offset from the plan's element 0
};
static_assert(sizeof(Seg) == 24, "Seg layout is mirrored by numpy in parallel/plan.py");

// ---- collectives.cu
void launch_plan(const CommCtx& ctx, int kind, int wire_dtype, bool nvls, int grid, const std::vector<at::Tensor>& tensors,
                 int64_t seg_begin_ptr, int64_t segs_ptr, int64_t data_off_bytes, int64_t block_elems, int64_t plan_calls_ptr,
                 int64_t found_inf_ptr, double scale, bool writeback, int root, int flags = 0, int64_t result_off_bytes = -1);
at::Tensor pack_pointers(const std::vector<at::Tensor>& tensors);
// rank-local fp32 gradient accumulation over one bucket's plan: acc[acc_off + seg.arena_off + i] += g (fold=false), or
// g = round(acc + g) and acc = 0 (fold=true); `split` CTAs share each plan CTA's segments
void grad_accum(const std::vector<at::Tensor>& grads, const at::Tensor& seg_begin, const at::Tensor& segs, int64_t grid, int64_t split,
                at::Tensor acc, int64_t acc_off, int64_t region_elems, bool fold);
void launch_barrier(const CommCtx& ctx);
void launch_metrics(const CommCtx& ctx, const at::Tensor& logits, const at::Tensor& target, const c10::optional<at::Tensor>& loss,
                    int64_t ll_seq_ptr, at::Tensor out);
void launch_ll_allreduce(const CommCtx& ctx, const at::Tensor& in, at::Tensor out, double scale, int64_t ll_seq_ptr);

// ---- optim.cu
// `ema` (optional, ModelEma): fp32 averages updated from the new masters with the decay in hyper[6], hyper[7]
void fused_sgd_flat(at::Tensor grad, at::Tensor master, at::Tensor momentum, c10::optional<at::Tensor> model_copy,
                    at::Tensor hyper, c10::optional<at::Tensor> found_inf, bool nesterov, bool first_step, c10::optional<at::Tensor> ema);
void fused_sgd_multi(std::vector<at::Tensor> grads, std::vector<at::Tensor> params, std::vector<at::Tensor> momenta,
                     std::vector<at::Tensor> model_copies, at::Tensor hyper, c10::optional<at::Tensor> found_inf, bool nesterov,
                     bool first_step, std::vector<at::Tensor> ema);
// dst = fmaf(dw[0], dst, dw[1] * src) over tensor lists (fp32 dst), nothing when found_inf is set
void ema_multi(std::vector<at::Tensor> src, std::vector<at::Tensor> dst, at::Tensor dw, c10::optional<at::Tensor> found_inf);
void multi_tensor_scale(std::vector<at::Tensor> src, std::vector<at::Tensor> dst, double scale, at::Tensor found_inf);
void multi_tensor_axpby(std::vector<at::Tensor> x, std::vector<at::Tensor> y, std::vector<at::Tensor> out, double a, double b,
                        at::Tensor found_inf);
// LARC: norm pass + SGD update (flat: chunks [chunk_lo, chunk_hi) of a table built once per layout; multi: whole lists)
constexpr int64_t kLarcChunkElems = 8192;
void larc_sgd_flat(at::Tensor grad, at::Tensor master, at::Tensor momentum, c10::optional<at::Tensor> model_copy, at::Tensor hyper,
                   c10::optional<at::Tensor> found_inf, bool nesterov, bool first_step, at::Tensor chunk_tensor, at::Tensor info,
                   int64_t chunk_lo, int64_t chunk_hi, at::Tensor partials, at::Tensor stats, double trust, double eps, bool clip,
                   c10::optional<at::Tensor> ema);
void larc_sgd_multi(std::vector<at::Tensor> grads, std::vector<at::Tensor> params, std::vector<at::Tensor> momenta,
                    std::vector<c10::optional<at::Tensor>> model_copies, at::Tensor hyper, c10::optional<at::Tensor> found_inf, bool nesterov,
                    std::vector<bool> first, std::vector<int64_t> rows, at::Tensor stats, double trust, double eps, bool clip,
                    std::vector<at::Tensor> ema);
// Global-norm clipping: per-chunk partials of sum (g * hyper[4])^2 (flat: the LARC chunk table; multi: partials
// [partial_off, returned value) of one buffer shared by every launch of a step), then one CTA forming the norm into `total`,
// the clipped hyper copies (slot 4 times min(hyper[8] / (norm + 1e-6), 1)) and `count` += (coef < 1)
void grad_sumsq_flat(at::Tensor grad, at::Tensor chunk_tensor, at::Tensor info, at::Tensor partials, at::Tensor hyper,
                     c10::optional<at::Tensor> found_inf);
int64_t grad_sumsq_multi(std::vector<at::Tensor> grads, at::Tensor hyper, c10::optional<at::Tensor> found_inf, at::Tensor partials,
                         int64_t partial_off);
void clip_finalize(at::Tensor partials, int64_t nparts, std::vector<at::Tensor> hypers, std::vector<at::Tensor> clipped,
                   c10::optional<at::Tensor> found_inf, at::Tensor total, at::Tensor count);
void amp_update_scale(at::Tensor scale, at::Tensor growth_tracker, at::Tensor found_inf, double growth, double backoff,
                      int64_t interval, at::Tensor hyper);

// ---- bn_act.cu
// gsum[0:n] += the rows part[0:nblocks][0:n] summed in a fixed order (deterministic cross-CTA reduction)
void combine_partials(const float* part, int nblocks, int n, float* gsum, cudaStream_t st);
// The entry points below take `sync` (nullptr: this rank alone).  With a handle, `work` is the synchronised layout
// float[kSyncWork(C)] = [local 2C sums | global 2C sums | global row count (int64)] instead of the plain [2C] sums.
std::vector<at::Tensor> bn_act_forward(const at::Tensor& x, const c10::optional<at::Tensor>& residual, const at::Tensor& weight,
                                       const at::Tensor& bias, at::Tensor running_mean, at::Tensor running_var,
                                       c10::optional<at::Tensor> num_batches_tracked, bool training, double momentum, double eps, bool relu,
                                       bool need_mask, at::Tensor work, bool stats_ready, const SyncBN* sync);
std::vector<at::Tensor> bn_act_backward(const at::Tensor& dy, const at::Tensor& x, const c10::optional<at::Tensor>& mask,
                                        const at::Tensor& weight, const at::Tensor& saved, bool relu, bool has_residual, at::Tensor work,
                                        const SyncBN* sync);
std::vector<at::Tensor> bn_act_backward2(const at::Tensor& dy_a, const at::Tensor& dy_b, const at::Tensor& x,
                                         const c10::optional<at::Tensor>& mask, const at::Tensor& weight, const at::Tensor& saved, bool relu,
                                         at::Tensor work, const SyncBN* sync);
// The backward of a 1x1 conv -> BatchNorm pair of one rank: the reduction pass, then gemm_bnstats.cu's data-gradient GEMM that
// applies the BatchNorm backward to its A operand.  returns {d conv input, dx, g (with dy_b), dweight, dbias}
std::vector<at::Tensor> conv1x1_bn_backward(const at::Tensor& dy_a, const c10::optional<at::Tensor>& dy_b, const at::Tensor& y,
                                            const c10::optional<at::Tensor>& mask, const at::Tensor& weight, const at::Tensor& saved,
                                            const at::Tensor& conv_weight, bool relu, at::Tensor work);

std::vector<at::Tensor> stem_forward(const at::Tensor& x, const at::Tensor& weight, const at::Tensor& bias, at::Tensor running_mean,
                                     at::Tensor running_var, c10::optional<at::Tensor> num_batches_tracked, bool training, double momentum,
                                     double eps, bool need_code, at::Tensor work, const SyncBN* sync);
std::vector<at::Tensor> stem_forward_pre(const at::Tensor& x, const at::Tensor& weight, const at::Tensor& bias, at::Tensor running_mean,
                                         at::Tensor running_var, c10::optional<at::Tensor> num_batches_tracked, bool training, double momentum,
                                         double eps, bool need_code, at::Tensor work, const SyncBN* sync);
std::vector<at::Tensor> stem_backward(const at::Tensor& dp, const at::Tensor& x, const at::Tensor& code, const at::Tensor& weight,
                                      const at::Tensor& saved, at::Tensor work, const SyncBN* sync);

// ---- sync_bn.cu
// floats of a synchronised work slice for C channels (the int64 count stays 8-byte aligned: C % 8 == 0)
constexpr int64_t kSyncWork(int64_t C) { return 4 * C + 4; }
// Replaces combine_partials for a synchronised layer: work[0:2C] += the fixed-order combine of part (this rank's sums),
// then every rank publishes them with its row count and work[2C:4C] / work[4C:4C+2] receive the rank-order global sums
// and the global count.
void sync_bn_exchange(const float* part, int nblocks, int C, int64_t rows, float* work, const SyncBN& s, cudaStream_t st);
// `work` is a float work slice of one direction of a C-channel layer: [2C], or [kSyncWork(C)] with a handle
void check_work(const at::Tensor& work, int64_t C, const SyncBN* sync);
// Where an apply kernel reads its sums in a work slice: the global sums with a handle, else this rank's
float* work_sums(float* work, int C, const SyncBN* sync);
// The reduction step after every pass that wrote per-CTA partials: sync_bn_exchange with a handle, else combine_partials.
// Returns work_sums(work, C, sync).
float* finish_sums(const float* part, int nblocks, int C, int64_t rows, float* work, const SyncBN* sync, cudaStream_t st);

// ---- gemm_bnstats.cu (wgmma / TMA)
at::Tensor conv1x1_bnstats(const at::Tensor& x, const at::Tensor& weight, at::Tensor gsum, const SyncBN* sync);
// dIn = dx x W with dx = bn_bwd_dx(A, B, D, g (x mask bits), y) formed in shared memory and also written to `dx`; A / B / D
// from saved, sums and bnw (dtype wdt), which block 0 also writes as dw / db (as bn_bwd_apply does).  mask: nullptr, or the
// forward's ReLU bits.  conv_w: [K, N, 1, 1], dx: [M, K], din: [M, N], all channels_last.
void conv1x1_dgrad_bn(const at::Tensor& g, const at::Tensor& y, const uint8_t* mask, const at::Tensor& saved, const float* sums,
                      const at::Tensor& bnw, int wdt, at::Tensor& dw, at::Tensor& db, const at::Tensor& conv_w, at::Tensor& dx, at::Tensor& din);

// ---- stem_conv.cu
at::Tensor stem_im2col(const at::Tensor& x);

// ---- data_ops.cu
at::Tensor normalize_nhwc(const at::Tensor& src, const at::Tensor& mean, const at::Tensor& std, int64_t out_dtype, bool channels_last);

void p2p_copy_multi(std::vector<at::Tensor> src, std::vector<at::Tensor> dst, int64_t run_device);

// ---- resample.cu (out_dtype kU8Out: the rounded uint8 pixels, NCHW, without the normalisation)
constexpr int64_t kU8Out = 3;
at::Tensor resample_normalize(const at::Tensor& arena, int64_t n, int64_t out_h, int64_t out_w, int64_t max_rows, const at::Tensor& a,
                              const at::Tensor& b, int64_t out_dtype, bool channels_last);

// ---- mix.cu (prm: the float[8] per-step parameters, see mix.cu)
// out = MixUp / CutMix of x with roll(x, 1, 0); yb = roll(y, 1); dom = the argmax label of the mixed target
void mix_batch(const at::Tensor& x, at::Tensor out, const at::Tensor& y, at::Tensor yb, at::Tensor dom, const at::Tensor& prm);
// cross-entropy against (1-eps)(la onehot(ya) + lb onehot(yb)) + eps/C: returns {mean loss, per-row loss, per-row lse}
std::vector<at::Tensor> soft_ce_fwd(const at::Tensor& z, const at::Tensor& ya, const at::Tensor& yb, const at::Tensor& prm, double eps);
// dz = g[0] / B (softmax(z) - q), in the logits' dtype
at::Tensor soft_ce_bwd(const at::Tensor& z, const at::Tensor& ya, const at::Tensor& yb, const at::Tensor& prm, const at::Tensor& lse,
                       const at::Tensor& g, double eps);

// ---- augment.cu (prm: float32 [n, kAugPrm] or [n, kAugChainPrm], one row of encoded op parameters per sample, see augment.cu)
// TrivialAugmentWide or AutoAugment + normalise + RandomErasing of a uint8 NCHW batch; returns what normalize_nhwc returns for
// it unaugmented
constexpr int64_t kAugPrm = 16;               // one op per sample
constexpr int64_t kAugChainPrm = 32;          // two ops per sample, the second applied to the first's output
constexpr int64_t kAugMaxPixels = 65793;      // 255 H W < 2^24: Contrast's float32 grayscale sum is exact in any order
at::Tensor augment_normalize(const at::Tensor& src, const at::Tensor& prm, const at::Tensor& a, const at::Tensor& b, int64_t out_dtype,
                             bool channels_last);

}  // namespace ptd
