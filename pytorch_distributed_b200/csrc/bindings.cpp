// Python bindings for the native runtime (pybind11 through torch/extension.h).
#include <torch/extension.h>

#include "hvd_core.h"
#include "host.h"
#include "symm.h"

namespace py = pybind11;
using namespace ptd;

namespace {

at::Tensor arena_view(const std::shared_ptr<SymmArena>& a, int64_t rank, int64_t offset_bytes, int64_t numel, const std::string& dtype) {
  at::ScalarType st;
  if (dtype == "float32") st = at::kFloat;
  else if (dtype == "bfloat16") st = at::kBFloat16;
  else if (dtype == "float16") st = at::kHalf;
  else if (dtype == "int32") st = at::kInt;
  else if (dtype == "uint8") st = at::kByte;
  else throw std::runtime_error("unsupported arena view dtype " + dtype);
  const int64_t esz = (int64_t)c10::elementSize(st);
  TORCH_CHECK(offset_bytes >= 0 && offset_bytes + numel * esz <= a->bytes(), "arena view out of range");
  TORCH_CHECK(offset_bytes % esz == 0, "misaligned arena view");
  const int r = a->single_process() ? (int)rank : a->rank();
  void* p = reinterpret_cast<void*>(a->ptr(r) + offset_bytes);
  auto keep = a;  // the tensor keeps the arena alive
  return at::from_blob(p, {numel}, [keep](void*) {}, at::TensorOptions().dtype(st).device(at::kCUDA, (c10::DeviceIndex)a->device(r)));
}

}  // namespace

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.doc() = "pytorch_distributed_b200 native runtime (sm_90a)";
  m.attr("MAX_WORLD") = kMaxWorld;
  m.attr("MAX_BLOCKS") = kMaxBlocks;
  m.attr("MAX_CHANNELS") = kMaxChannels;
  m.attr("MAX_PTRS") = kMaxPtrs;
  m.attr("SIGNAL_PAD_BYTES") = (int64_t)sizeof(SignalPad);
  m.attr("SEG_BYTES") = (int64_t)sizeof(Seg);
  m.attr("SYNC_BN_MAX_C") = kSyncBnMaxC;
  m.attr("SYNC_BN_AREA_BYTES") = kSyncBnAreaBytes;
  m.def("multicast_supported", &multicast_supported);

  // handle of a synchronised BatchNorm layer group: the peers' context, the exchange area offset, the call counters
  py::class_<SyncBN>(m, "SyncBN")
      .def_property_readonly("rank", [](const SyncBN& s) { return s.ctx.rank; })
      .def_property_readonly("world", [](const SyncBN& s) { return s.ctx.world; })
      .def_property_readonly("xoff", [](const SyncBN& s) { return s.xoff; });

  py::class_<SymmArena, std::shared_ptr<SymmArena>>(m, "SymmArena")
      .def(py::init<int, int, int, int64_t>(), py::arg("device"), py::arg("rank"), py::arg("world"), py::arg("bytes"))
      .def_static("create_local", &SymmArena::create_local)
      .def_static("from_pointers", &SymmArena::from_pointers)
      .def("export_fd", &SymmArena::export_fd)
      .def("open_socket", &SymmArena::open_socket)
      .def("send_fd", &SymmArena::send_fd)
      .def("recv_fd", &SymmArena::recv_fd, py::call_guard<py::gil_scoped_release>())
      .def("map_peer", &SymmArena::map_peer)
      .def("mc_create", &SymmArena::mc_create)
      .def("mc_import", &SymmArena::mc_import)
      .def("mc_add_device", &SymmArena::mc_add_device)
      .def("mc_bind_and_map", &SymmArena::mc_bind_and_map)
      .def("disable_multicast", &SymmArena::disable_multicast)
      .def_property_readonly("rank", &SymmArena::rank)
      .def_property_readonly("world", &SymmArena::world)
      .def_property_readonly("bytes", &SymmArena::bytes)
      .def_property_readonly("mc_ptr", &SymmArena::mc_ptr)
      .def_property_readonly("multicast_candidate", &SymmArena::multicast_candidate)
      .def_property_readonly("has_multicast", &SymmArena::has_multicast)
      .def_property_readonly("mc_error", &SymmArena::mc_error)
      .def_property_readonly("single_process", &SymmArena::single_process)
      .def("ptr", &SymmArena::ptr)
      .def("device", &SymmArena::device, py::arg("r") = 0)
      .def("status", &SymmArena::status)
      .def("set_timeout_ms", &SymmArena::set_timeout_ms)
      .def("ll_seq_ptr", &SymmArena::ll_seq_ptr, py::arg("r") = 0)
      .def("view", [](std::shared_ptr<SymmArena> a, int64_t offset, int64_t numel, const std::string& dtype, int64_t rank) {
             return arena_view(a, rank, offset, numel, dtype);
           }, py::arg("offset_bytes"), py::arg("numel"), py::arg("dtype"), py::arg("rank") = 0)
      .def("launch_plan",
           [](std::shared_ptr<SymmArena> a, int channel, int as_rank, int kind, int wire_dtype, bool nvls, int grid, std::vector<at::Tensor> tensors,
              int64_t seg_begin_ptr, int64_t segs_ptr, int64_t data_off_bytes, int64_t block_elems, int64_t plan_calls_ptr, int64_t found_inf_ptr,
              double scale, bool writeback, int root, int flags, int64_t result_off_bytes) {
             launch_plan(a->ctx(channel, as_rank), kind, wire_dtype, nvls, grid, tensors, seg_begin_ptr, segs_ptr, data_off_bytes, block_elems,
                         plan_calls_ptr, found_inf_ptr, scale, writeback, root, flags, result_off_bytes);
           },
           py::arg("channel"), py::arg("as_rank"), py::arg("kind"), py::arg("wire_dtype"), py::arg("nvls"), py::arg("grid"), py::arg("tensors"),
           py::arg("seg_begin_ptr"), py::arg("segs_ptr"), py::arg("data_off_bytes"), py::arg("block_elems"), py::arg("plan_calls_ptr"),
           py::arg("found_inf_ptr"), py::arg("scale"), py::arg("writeback"), py::arg("root"), py::arg("flags") = 0,
           py::arg("result_off_bytes") = (int64_t)-1)
      .def("launch_barrier", [](std::shared_ptr<SymmArena> a, int channel) { launch_barrier(a->ctx(channel)); })
      .def("launch_metrics",
           [](std::shared_ptr<SymmArena> a, int channel, const at::Tensor& logits, const at::Tensor& target, c10::optional<at::Tensor> loss, at::Tensor out) {
             launch_metrics(a->ctx(channel), logits, target, loss, a->ll_seq_ptr(), out);
           })
      .def("launch_ll_allreduce", [](std::shared_ptr<SymmArena> a, int channel, const at::Tensor& in, at::Tensor out, double scale) {
        launch_ll_allreduce(a->ctx(channel), in, out, scale, a->ll_seq_ptr());
      })
      .def("sync_bn",
           [](std::shared_ptr<SymmArena> a, int channel, int64_t xoff, int64_t calls_ptr, int as_rank) {
             TORCH_CHECK(xoff >= 0 && xoff % 16 == 0 && xoff + kSyncBnAreaBytes <= a->bytes(), "sync BN exchange area outside the arena");
             TORCH_CHECK(calls_ptr != 0, "sync BN call counters missing");
             return SyncBN{a->ctx(channel, as_rank), xoff, reinterpret_cast<uint32_t*>(calls_ptr)};
           },
           py::arg("channel"), py::arg("xoff"), py::arg("calls_ptr"), py::arg("as_rank") = 0);

  m.def("pack_pointers", &pack_pointers);
  m.def("grad_accumulate",
        [](const std::vector<at::Tensor>& grads, const at::Tensor& seg_begin, const at::Tensor& segs, int64_t grid, int64_t split, at::Tensor acc,
           int64_t acc_off, int64_t region_elems) { grad_accum(grads, seg_begin, segs, grid, split, acc, acc_off, region_elems, false); },
        py::arg("grads"), py::arg("seg_begin"), py::arg("segs"), py::arg("grid"), py::arg("split"), py::arg("acc"), py::arg("acc_off"),
        py::arg("region_elems"));
  m.def("grad_fold",
        [](const std::vector<at::Tensor>& grads, const at::Tensor& seg_begin, const at::Tensor& segs, int64_t grid, int64_t split, at::Tensor acc,
           int64_t acc_off, int64_t region_elems) { grad_accum(grads, seg_begin, segs, grid, split, acc, acc_off, region_elems, true); },
        py::arg("grads"), py::arg("seg_begin"), py::arg("segs"), py::arg("grid"), py::arg("split"), py::arg("acc"), py::arg("acc_off"),
        py::arg("region_elems"));
  m.def("fused_sgd_flat", &fused_sgd_flat, py::arg("grad"), py::arg("master"), py::arg("momentum"), py::arg("model_copy"), py::arg("hyper"),
        py::arg("found_inf"), py::arg("nesterov"), py::arg("first_step"), py::arg("ema") = c10::optional<at::Tensor>());
  m.def("fused_sgd_multi", &fused_sgd_multi, py::arg("grads"), py::arg("params"), py::arg("momenta"), py::arg("model_copies"),
        py::arg("hyper"), py::arg("found_inf"), py::arg("nesterov"), py::arg("first_step"), py::arg("ema") = std::vector<at::Tensor>());
  m.def("ema_multi", &ema_multi, py::arg("src"), py::arg("dst"), py::arg("dw"), py::arg("found_inf") = c10::optional<at::Tensor>());
  m.attr("LARC_CHUNK") = kLarcChunkElems;
  m.def("larc_sgd_flat", &larc_sgd_flat, py::arg("grad"), py::arg("master"), py::arg("momentum"), py::arg("model_copy"), py::arg("hyper"),
        py::arg("found_inf"), py::arg("nesterov"), py::arg("first_step"), py::arg("chunk_tensor"), py::arg("info"), py::arg("chunk_lo"),
        py::arg("chunk_hi"), py::arg("partials"), py::arg("stats"), py::arg("trust"), py::arg("eps"), py::arg("clip"),
        py::arg("ema") = c10::optional<at::Tensor>());
  m.def("larc_sgd_multi", &larc_sgd_multi, py::arg("grads"), py::arg("params"), py::arg("momenta"), py::arg("model_copies"), py::arg("hyper"),
        py::arg("found_inf"), py::arg("nesterov"), py::arg("first"), py::arg("rows"), py::arg("stats"), py::arg("trust"), py::arg("eps"),
        py::arg("clip"), py::arg("ema") = std::vector<at::Tensor>());
  m.def("grad_sumsq_flat", &grad_sumsq_flat, py::arg("grad"), py::arg("chunk_tensor"), py::arg("info"), py::arg("partials"),
        py::arg("hyper"), py::arg("found_inf"));
  m.def("grad_sumsq_multi", &grad_sumsq_multi, py::arg("grads"), py::arg("hyper"), py::arg("found_inf"), py::arg("partials"),
        py::arg("partial_off"));
  m.def("clip_finalize", &clip_finalize, py::arg("partials"), py::arg("nparts"), py::arg("hypers"), py::arg("clipped"), py::arg("found_inf"),
        py::arg("total"), py::arg("count"));
  m.def("multi_tensor_scale", &multi_tensor_scale);
  m.def("multi_tensor_axpby", &multi_tensor_axpby);
  m.def("amp_update_scale", &amp_update_scale);
  // BatchNorm entry points: `sync` (a SyncBN, default None = this rank alone) selects the synchronised variant
  const auto sync_arg = py::arg("sync") = static_cast<const SyncBN*>(nullptr);
  m.def("bn_act_forward", &bn_act_forward, py::arg("x"), py::arg("residual"), py::arg("weight"), py::arg("bias"), py::arg("running_mean"),
        py::arg("running_var"), py::arg("num_batches_tracked"), py::arg("training"), py::arg("momentum"), py::arg("eps"), py::arg("relu"),
        py::arg("need_mask"), py::arg("work"), py::arg("stats_ready"), sync_arg);
  m.def("bn_act_backward", &bn_act_backward, py::arg("dy"), py::arg("x"), py::arg("mask"), py::arg("weight"), py::arg("saved"), py::arg("relu"),
        py::arg("has_residual"), py::arg("work"), sync_arg);
  m.def("bn_act_backward2", &bn_act_backward2, py::arg("dy_a"), py::arg("dy_b"), py::arg("x"), py::arg("mask"), py::arg("weight"),
        py::arg("saved"), py::arg("relu"), py::arg("work"), sync_arg);
  m.def("stem_forward", &stem_forward, py::arg("x"), py::arg("weight"), py::arg("bias"), py::arg("running_mean"), py::arg("running_var"),
        py::arg("num_batches_tracked"), py::arg("training"), py::arg("momentum"), py::arg("eps"), py::arg("need_code"), py::arg("work"), sync_arg);
  m.def("stem_forward_pre", &stem_forward_pre, py::arg("x"), py::arg("weight"), py::arg("bias"), py::arg("running_mean"), py::arg("running_var"),
        py::arg("num_batches_tracked"), py::arg("training"), py::arg("momentum"), py::arg("eps"), py::arg("need_code"), py::arg("work"), sync_arg);
  m.def("stem_backward", &stem_backward, py::arg("dp"), py::arg("x"), py::arg("code"), py::arg("weight"), py::arg("saved"), py::arg("work"),
        sync_arg);
  m.def("stem_im2col", &stem_im2col);
  m.def("conv1x1_bnstats", &conv1x1_bnstats, py::arg("x"), py::arg("weight"), py::arg("gsum"), sync_arg);
  m.def("conv1x1_bn_backward", &conv1x1_bn_backward, py::arg("dy_a"), py::arg("dy_b"), py::arg("y"), py::arg("mask"), py::arg("weight"),
        py::arg("saved"), py::arg("conv_weight"), py::arg("relu"), py::arg("work"));
  m.def("normalize_nhwc", &normalize_nhwc);
  m.def("resample_normalize", &resample_normalize, py::arg("arena"), py::arg("n"), py::arg("out_h"), py::arg("out_w"), py::arg("max_rows"),
        py::arg("a"), py::arg("b"), py::arg("out_dtype"), py::arg("channels_last"));
  m.attr("U8_OUT") = kU8Out;
  m.def("augment_normalize", &augment_normalize, py::arg("src"), py::arg("prm"), py::arg("a"), py::arg("b"), py::arg("out_dtype"),
        py::arg("channels_last"));
  m.attr("AUG_PRM") = kAugPrm;
  m.attr("AUG_CHAIN_PRM") = kAugChainPrm;
  m.attr("AUG_MAX_PIXELS") = kAugMaxPixels;
  m.def("p2p_copy_multi", &p2p_copy_multi);
  m.def("mix_batch", &mix_batch, py::arg("x"), py::arg("out"), py::arg("y"), py::arg("yb"), py::arg("dom"), py::arg("prm"));
  m.def("soft_ce_fwd", &soft_ce_fwd, py::arg("z"), py::arg("ya"), py::arg("yb"), py::arg("prm"), py::arg("eps"));
  m.def("soft_ce_bwd", &soft_ce_bwd, py::arg("z"), py::arg("ya"), py::arg("yb"), py::arg("prm"), py::arg("lse"), py::arg("g"), py::arg("eps"));

  // horovod-style fusion queue (background thread + tensor fusion scheduling), see hvd_core.cpp
  py::class_<FusionQueue, std::shared_ptr<FusionQueue>>(m, "FusionQueue")
      .def(py::init<int64_t, double, int64_t>(), py::arg("fusion_threshold_bytes"), py::arg("cycle_time_ms"), py::arg("cycle_bytes") = 0)
      .def("wait_idle", &FusionQueue::wait_idle, py::arg("timeout_ms"), py::call_guard<py::gil_scoped_release>())
      .def("wake", &FusionQueue::wake)
      .def("set_cycle_bytes", &FusionQueue::set_cycle_bytes)
      .def("cycle_bytes", &FusionQueue::cycle_bytes)
      .def("enable_timeline", &FusionQueue::enable_timeline)
      .def("timeline", &FusionQueue::timeline)
      .def("enqueue", &FusionQueue::enqueue, py::arg("name"), py::arg("nbytes"), py::arg("order_key"))
      .def("next_group", &FusionQueue::next_group, py::arg("timeout_ms"), py::call_guard<py::gil_scoped_release>())
      .def("flush", &FusionQueue::flush)
      .def("mark_done", &FusionQueue::mark_done)
      .def("wait", &FusionQueue::wait, py::arg("handle"), py::arg("timeout_ms"), py::call_guard<py::gil_scoped_release>())
      .def("pending", &FusionQueue::pending)
      .def("shutdown", &FusionQueue::shutdown)
      .def("stats", &FusionQueue::stats);
}
