// Native input pipeline: memory-mapped shards of pre-decoded uint8 images -> random-resized-crop / centre-crop,
// antialiased bilinear resample, horizontal flip -> planar uint8 batches written straight into (pinned) ring slots.
//
// Role: the reference feeds its loops with torch DataLoader worker PROCESSES running PIL per sample
// (reference distributed.py:160-195, transforms at :165-172 and :183-188).  At thousands of images/s per GPU that host
// path cannot keep a node busy, so the steady-state loader here is native: no Python, no pickling, no per-sample
// allocation in the hot loop.  JPEG decoding happens once, offline (tools/make_shards.py).  The device side is the
// existing fused normalise/cast/NHWC kernel (csrc/data_ops.cu), fed with the uint8 NCHW batches produced here.  In
// staging mode (Config::staged) the threads leave the resample to the GPU (csrc/resample.cu) and write, per sample, the
// source pixels and filter taps it needs instead.
//
// Determinism: the epoch permutation and every per-sample random decision are pure functions of
// (seed, epoch, position in the epoch), so results do not depend on thread scheduling or thread count.
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <condition_variable>
#include <cstdint>
#include <cstring>
#include <memory>
#include <mutex>
#include <stdexcept>
#include <string>
#include <thread>
#include <vector>

namespace py = pybind11;

namespace {

constexpr char kMagic[8] = {'P', 'T', 'D', 'S', 'H', 'R', 'D', '1'};

struct IndexEntry {        // 24 bytes, little endian, directly after the 16-byte header
  uint64_t offset;         // of the first pixel, from the start of the file
  uint32_t height, width;
  int32_t label;
  uint32_t channels;       // always 3
};
static_assert(sizeof(IndexEntry) == 24, "index entry layout");

struct Record {
  const uint8_t* px;
  uint32_t h, w;
  int32_t label;
};

// ---------------------------------------------------------------- counter-based RNG (splitmix64)
struct Rng {
  uint64_t s;
  explicit Rng(uint64_t seed) : s(seed) {}
  uint64_t next() {
    uint64_t z = (s += 0x9E3779B97F4A7C15ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
  }
  double uniform() { return (next() >> 11) * (1.0 / 9007199254740992.0); }      // [0, 1)
  double uniform(double lo, double hi) { return lo + (hi - lo) * uniform(); }
  uint64_t below(uint64_t n) { return n ? next() % n : 0; }                      // n << 2^64: bias is negligible
};

uint64_t mix(uint64_t a, uint64_t b, uint64_t c) {
  Rng r(a * 0xD6E8FEB86659FD93ull + b * 0xA5CB9243F1D1E7ABull + c + 0x632BE59BD9B4E019ull);
  r.next();
  return r.next();
}

// ---------------------------------------------------------------- crop boxes
struct Box { double x0, y0, w, h; bool clamp; bool flip; };

// torchvision.transforms.RandomResizedCrop.get_params: 10 tries of (area fraction, log-uniform aspect), then the
// largest centred crop whose aspect is inside the allowed range.
Box random_resized_crop(Rng& rng, int W, int H, double s_lo, double s_hi, double r_lo, double r_hi) {
  const double area = double(W) * H;
  const double lr_lo = std::log(r_lo), lr_hi = std::log(r_hi);
  for (int attempt = 0; attempt < 10; ++attempt) {
    const double target = area * rng.uniform(s_lo, s_hi);
    const double ratio = std::exp(rng.uniform(lr_lo, lr_hi));
    const int w = int(std::lround(std::sqrt(target * ratio)));
    const int h = int(std::lround(std::sqrt(target / ratio)));
    if (w > 0 && w <= W && h > 0 && h <= H) {
      const int y = int(rng.below(uint64_t(H - h + 1)));
      const int x = int(rng.below(uint64_t(W - w + 1)));
      return {double(x), double(y), double(w), double(h), true, false};
    }
  }
  const double in_ratio = double(W) / H;
  int w = W, h = H;
  if (in_ratio < r_lo) { h = int(std::lround(W / r_lo)); }
  else if (in_ratio > r_hi) { w = int(std::lround(H * r_hi)); }
  w = std::max(1, std::min(w, W));
  h = std::max(1, std::min(h, H));
  return {double((W - w) / 2), double((H - h) / 2), double(w), double(h), true, false};
}

// Resize(shorter side -> out * resize_ratio) followed by CenterCrop(out), expressed as one box in source coordinates.
// The filter may read pixels outside the box (as resize-then-crop does), hence clamp = false.
Box center_crop(int W, int H, int out_w, int out_h, double resize_ratio) {
  // Integer geometry exactly as torchvision computes it: the resized image is rw x rh (shorter side S, longer side
  // truncated), the crop starts at round-half-even((r - out) / 2).
  const int S = std::max(1, int(std::max(out_w, out_h) * resize_ratio + 1e-9));     // e.g. 256 for out = 224
  int rw, rh;
  if (W <= H) { rw = S; rh = std::max(1, int(double(S) * H / W)); }
  else        { rh = S; rw = std::max(1, int(double(S) * W / H)); }
  const double sx = double(W) / rw, sy = double(H) / rh;                // source pixels per resized pixel
  const double left = std::max(0.0, std::nearbyint((rw - out_w) / 2.0));
  const double top = std::max(0.0, std::nearbyint((rh - out_h) / 2.0));
  const double bw = std::min(double(out_w), double(rw)) * sx, bh = std::min(double(out_h), double(rh)) * sy;
  return {left * sx, top * sy, bw, bh, false, false};
}

// ---------------------------------------------------------------- antialiased bilinear resample (triangle filter)
struct Taps {
  std::vector<int> first, count;     // per output coordinate
  std::vector<float> weight;         // [out][kmax]
  int kmax = 0;
};

// Same construction as Pillow's precompute_coeffs / ATen's antialiased bilinear kernel: support widens with the
// down-scaling factor, taps are clipped to [lo, hi) and renormalised.
void build_taps(Taps& t, int out, double in0, double in_len, int lo, int hi, bool reverse) {
  const double scale = in_len / out;
  const double fscale = std::max(scale, 1.0);
  const double support = fscale;                      // triangle filter has support 1
  t.kmax = int(std::ceil(support)) * 2 + 1;
  t.first.assign(out, 0);
  t.count.assign(out, 0);
  t.weight.assign(size_t(out) * t.kmax, 0.f);
  for (int o = 0; o < out; ++o) {
    const int src_o = reverse ? out - 1 - o : o;
    const double center = in0 + (src_o + 0.5) * scale;
    int xmin = int(center - support + 0.5);
    int xmax = int(center + support + 0.5);
    xmin = std::max(xmin, lo);
    xmax = std::min(xmax, hi);
    int n = std::max(0, xmax - xmin);
    if (n == 0) {                                     // degenerate (box at the border): nearest valid pixel
      xmin = std::min(std::max(int(center), lo), hi - 1);
      n = 1;
    }
    n = std::min(n, t.kmax);
    float* w = &t.weight[size_t(o) * t.kmax];
    double total = 0.0;
    for (int k = 0; k < n; ++k) {
      const double x = (xmin + k - center + 0.5) / fscale;
      const double v = std::max(0.0, 1.0 - std::fabs(x));
      w[k] = float(v);
      total += v;
    }
    if (total <= 0.0) { w[0] = 1.f; total = 1.0; for (int k = 1; k < n; ++k) w[k] = 0.f; }
    const float inv = float(1.0 / total);
    for (int k = 0; k < n; ++k) w[k] *= inv;
    t.first[o] = xmin;
    t.count[o] = n;
  }
}

struct Scratch {
  Taps tx, ty;
  std::vector<float> rows;       // horizontally resampled rows [n_rows][out_w][3]
};

// [lo, hi) of the source coordinates the taps read
std::pair<int, int> tap_span(const Taps& t) {
  int lo = INT32_MAX, hi = 0;
  for (size_t o = 0; o < t.first.size(); ++o) {
    lo = std::min(lo, t.first[o]);
    hi = std::max(hi, t.first[o] + t.count[o]);
  }
  return {lo, hi};
}

void build_box_taps(Scratch& s, int W, int H, const Box& b, int out_w, int out_h) {
  const int lo_x = b.clamp ? int(b.x0) : 0, hi_x = b.clamp ? int(b.x0 + b.w) : W;
  const int lo_y = b.clamp ? int(b.y0) : 0, hi_y = b.clamp ? int(b.y0 + b.h) : H;
  build_taps(s.tx, out_w, b.x0, b.w, lo_x, std::min(hi_x, W), b.flip);
  build_taps(s.ty, out_h, b.y0, b.h, lo_y, std::min(hi_y, H), false);
}

// src: HWC uint8 (H x W x 3).  dst: planar CHW uint8 (3 x out_h x out_w).
void resample(const Record& r, const Box& b, int out_w, int out_h, uint8_t* dst, Scratch& s) {
  const int W = int(r.w);
  build_box_taps(s, W, int(r.h), b, out_w, out_h);
  const auto [y_first, y_last] = tap_span(s.ty);
  const int n_rows = y_last - y_first;
  s.rows.resize(size_t(n_rows) * out_w * 3);
  const int kx = s.tx.kmax;
  for (int y = 0; y < n_rows; ++y) {                                     // horizontal pass
    const uint8_t* src = r.px + size_t(y_first + y) * W * 3;
    float* out = &s.rows[size_t(y) * out_w * 3];
    for (int o = 0; o < out_w; ++o) {
      const uint8_t* p = src + size_t(s.tx.first[o]) * 3;
      const float* w = &s.tx.weight[size_t(o) * kx];
      float a0 = 0.f, a1 = 0.f, a2 = 0.f;
      const int n = s.tx.count[o];
      for (int k = 0; k < n; ++k) {
        a0 += w[k] * p[3 * k];
        a1 += w[k] * p[3 * k + 1];
        a2 += w[k] * p[3 * k + 2];
      }
      out[3 * o] = a0; out[3 * o + 1] = a1; out[3 * o + 2] = a2;
    }
  }
  const int ky = s.ty.kmax;
  const size_t plane = size_t(out_h) * out_w;
  for (int o = 0; o < out_h; ++o) {                                      // vertical pass, planar output
    const float* w = &s.ty.weight[size_t(o) * ky];
    const int n = s.ty.count[o];
    const float* base = &s.rows[size_t(s.ty.first[o] - y_first) * out_w * 3];
    uint8_t* d0 = dst + size_t(o) * out_w;
    for (int x = 0; x < out_w; ++x) {
      float a0 = 0.f, a1 = 0.f, a2 = 0.f;
      for (int k = 0; k < n; ++k) {
        const float* p = base + (size_t(k) * out_w + x) * 3;
        a0 += w[k] * p[0]; a1 += w[k] * p[1]; a2 += w[k] * p[2];
      }
      d0[x] = uint8_t(std::min(255.f, std::max(0.f, a0 + 0.5f)));
      d0[plane + x] = uint8_t(std::min(255.f, std::max(0.f, a1 + 0.5f)));
      d0[2 * plane + x] = uint8_t(std::min(255.f, std::max(0.f, a2 + 0.5f)));
    }
  }
}

// ---------------------------------------------------------------- staging for the device resample
// In staging mode a worker does not call resample(): it copies the source rectangle the taps read, and the taps, into the
// slot's arena, and the GPU kernel (csrc/resample.cu) does resample()'s arithmetic.  Slot layout: `batch` StageDesc,
// then one 16-byte aligned block per sample, placed by a bump pointer: the region (rh x rw x 3 uint8, HWC), then the
// taps - x first (int32, relative to the region), x count (int32), x weights (float [out_w][kx]), and the same for y.
struct StageDesc {
  int64_t region;     // arena offset of the region
  int64_t taps;       // arena offset of the taps
  int32_t rw, rh;     // region width and height
  int32_t kx, ky;     // weights stored per output column / row
};
static_assert(sizeof(StageDesc) == 32, "StageDesc layout is mirrored in csrc/resample.cu and tests/test_cpu_device_resample.py");

constexpr size_t kStageAlign = 16;
size_t align_up(size_t v) { return (v + kStageAlign - 1) & ~(kStageAlign - 1); }
size_t taps_bytes(int out, int kmax) { return size_t(out) * (2 * sizeof(int32_t) + size_t(kmax) * sizeof(float)); }
size_t stage_bytes(int rw, int rh, int out_w, int kx, int out_h, int ky) {
  return align_up(size_t(rw) * rh * 3) + align_up(taps_bytes(out_w, kx) + taps_bytes(out_h, ky));
}
size_t table_bytes(int batch) { return align_up(size_t(batch) * sizeof(StageDesc)); }
int kmax_for(double in_len, int out) { return int(std::ceil(std::max(in_len / out, 1.0))) * 2 + 1; }   // as build_taps

uint8_t* put_taps(uint8_t* p, const Taps& t, int origin) {
  const size_t out = t.first.size();
  auto* first = reinterpret_cast<int32_t*>(p);
  auto* count = first + out;
  for (size_t o = 0; o < out; ++o) { first[o] = t.first[o] - origin; count[o] = t.count[o]; }
  std::memcpy(count + out, t.weight.data(), t.weight.size() * sizeof(float));
  return p + taps_bytes(int(out), t.kmax);
}

// ---------------------------------------------------------------- shard files
class Shard {
 public:
  explicit Shard(const std::string& path) {
    fd_ = ::open(path.c_str(), O_RDONLY);
    if (fd_ < 0) throw std::runtime_error("cannot open shard " + path);
    struct stat st;
    if (fstat(fd_, &st) != 0 || st.st_size < 16) { ::close(fd_); throw std::runtime_error("cannot stat shard " + path); }
    size_ = size_t(st.st_size);
    base_ = static_cast<const uint8_t*>(mmap(nullptr, size_, PROT_READ, MAP_SHARED, fd_, 0));
    if (base_ == MAP_FAILED) { ::close(fd_); throw std::runtime_error("cannot mmap shard " + path); }
    if (std::memcmp(base_, kMagic, 8) != 0) { unmap(); throw std::runtime_error("not a PTDSHRD1 shard: " + path); }
    uint32_t n;
    std::memcpy(&n, base_ + 8, 4);
    if (16 + size_t(n) * sizeof(IndexEntry) > size_) { unmap(); throw std::runtime_error("truncated shard index: " + path); }
    const auto* idx = reinterpret_cast<const IndexEntry*>(base_ + 16);
    records_.reserve(n);
    for (uint32_t i = 0; i < n; ++i) {
      const IndexEntry& e = idx[i];
      const size_t bytes = size_t(e.height) * e.width * 3;
      if (e.channels != 3 || e.height == 0 || e.width == 0 || e.offset + bytes > size_) {
        unmap();
        throw std::runtime_error("corrupt shard record in " + path);
      }
      records_.push_back({base_ + e.offset, e.height, e.width, e.label});
    }
  }
  ~Shard() { unmap(); }
  Shard(const Shard&) = delete;
  Shard& operator=(const Shard&) = delete;
  const std::vector<Record>& records() const { return records_; }

 private:
  void unmap() {
    if (base_ && base_ != MAP_FAILED) munmap(const_cast<uint8_t*>(base_), size_);
    if (fd_ >= 0) ::close(fd_);
    base_ = nullptr;
    fd_ = -1;
  }
  int fd_ = -1;
  size_t size_ = 0;
  const uint8_t* base_ = nullptr;
  std::vector<Record> records_;
};

struct Config {
  int batch, out_h, out_w;
  bool train;
  uint64_t seed;
  int rank, world, threads, depth;
  bool drop_last, shuffle;
  double scale_lo, scale_hi, ratio_lo, ratio_hi, resize_ratio;
  bool staged;          // stage regions + taps for the device resample instead of resampling on the host
};

// ---------------------------------------------------------------- the loader
class ShardLoader {
 public:
  ShardLoader(const std::vector<std::string>& paths, const Config& c) : cfg_(c) {
    if (c.batch <= 0 || c.out_h <= 0 || c.out_w <= 0 || c.world <= 0 || c.rank < 0 || c.rank >= c.world || c.depth < 2 ||
        c.threads <= 0)
      throw std::invalid_argument("bad ShardLoader configuration");
    for (const auto& p : paths) {
      shards_.emplace_back(new Shard(p));
      for (const auto& r : shards_.back()->records()) records_.push_back(r);
    }
    if (records_.empty()) throw std::runtime_error("no records in the given shards");
    const size_t n = records_.size();
    // DistributedSampler semantics: pad to a multiple of world by wrapping around, rank r takes positions r, r+world, ...
    per_rank_ = c.drop_last ? n / c.world : (n + c.world - 1) / c.world;
    if (per_rank_ == 0) throw std::runtime_error("fewer records than ranks with drop_last");
    n_batches_ = c.drop_last ? per_rank_ / c.batch : (per_rank_ + c.batch - 1) / c.batch;
    slot_done_.assign(c.depth, 0);
    stage_used_.reset(new std::atomic<size_t>[c.depth]);
    for (int s = 0; s < c.depth; ++s) stage_used_[s].store(0);
    if (c.staged) {
      std::vector<std::pair<uint32_t, uint32_t>> shapes;
      for (const auto& r : records_) shapes.emplace_back(r.w, r.h);
      std::sort(shapes.begin(), shapes.end());
      shapes.erase(std::unique(shapes.begin(), shapes.end()), shapes.end());
      size_t worst = 0;
      for (const auto& [W, H] : shapes) {
        worst = std::max(worst, stage_bound(int(W), int(H)));
        max_rows_ = std::max(max_rows_, rows_bound(int(W), int(H)));
      }
      stage_cap_ = table_bytes(c.batch) + size_t(c.batch) * worst;
    }
  }

  ~ShardLoader() { stop(); }

  size_t size() const { return records_.size(); }
  int64_t samples_per_rank() const { return int64_t(per_rank_); }
  int64_t num_batches() const { return int64_t(n_batches_); }
  int depth() const { return cfg_.depth; }

  void set_buffers(const std::vector<uintptr_t>& images, const std::vector<uintptr_t>& labels, const std::vector<uintptr_t>& ids) {
    if (int(images.size()) != cfg_.depth || int(labels.size()) != cfg_.depth || (!ids.empty() && int(ids.size()) != cfg_.depth))
      throw std::invalid_argument("need one buffer per ring slot");
    stop();
    images_ = images; labels_ = labels; ids_ = ids;
  }

  // Begin producing epoch `epoch`.  Any unfinished epoch is abandoned first.
  void start_epoch(int64_t epoch) {
    if (images_.empty()) throw std::runtime_error("set_buffers() first");
    stop();
    build_order(uint64_t(epoch));
    epoch_ = uint64_t(epoch);
    next_item_.store(0);
    consumed_ = 0;
    released_ = 0;
    std::fill(slot_done_.begin(), slot_done_.end(), 0);
    for (int s = 0; s < cfg_.depth; ++s) stage_used_[s].store(0);
    quit_ = false;
    for (int t = 0; t < cfg_.threads; ++t) workers_.emplace_back([this] { work(); });
  }

  // Blocks (GIL released by the binding) until the next batch is complete.  Returns {slot, batch_size} or {-1, 0}.
  std::pair<int, int> next() {
    if (consumed_ >= n_batches_) return {-1, 0};
    const size_t k = consumed_;
    const int slot = int(k % cfg_.depth);
    const int want = batch_size_of(k);
    std::unique_lock<std::mutex> lk(mu_);
    cv_done_.wait(lk, [&] { return slot_done_[slot] == want || !error_.empty(); });
    if (!error_.empty()) throw std::runtime_error(error_);
    ++consumed_;
    return {slot, want};
  }

  // The consumer is done with the oldest outstanding batch (its pinned slot may be overwritten).
  void release() {
    {
      std::lock_guard<std::mutex> lk(mu_);
      if (released_ >= consumed_) throw std::runtime_error("release() without a matching next()");
      slot_done_[released_ % cfg_.depth] = 0;
      stage_used_[released_ % cfg_.depth].store(0);
      ++released_;
    }
    cv_free_.notify_all();
  }

  void stop() {
    {
      std::lock_guard<std::mutex> lk(mu_);
      quit_ = true;
    }
    cv_free_.notify_all();
    for (auto& t : workers_) t.join();
    workers_.clear();
    error_.clear();
  }

  // test hook: the crop box sample `pos` of `epoch` gets for an image of the given size -> (x0, y0, w, h, flip)
  std::vector<double> crop_params(int64_t epoch, int64_t pos, int W, int H) const {
    Box b = box_for(uint64_t(epoch), uint64_t(pos), W, H);
    return {b.x0, b.y0, b.w, b.h, b.flip ? 1.0 : 0.0};
  }

  // test hook: record indices of this rank for `epoch`, in order
  std::vector<int64_t> epoch_order(int64_t epoch) {
    std::vector<uint32_t> keep;
    keep.swap(order_);
    build_order(uint64_t(epoch));
    std::vector<int64_t> out(order_.begin(), order_.end());
    order_.swap(keep);
    return out;
  }

  // ---- staging mode
  size_t stage_capacity() const { return stage_cap_; }      // bytes of one slot's arena
  int stage_max_rows() const { return max_rows_; }          // most source rows one output row reads, over all records
  // bytes of the arena in use by the batch next() returned last for `slot`
  size_t staged_bytes(int slot) const { return table_bytes(cfg_.batch) + stage_used_[slot].load(); }

  // Upper bound of the bytes one sample of a W x H record stages.  Train: the region lies inside the image and the box
  // is at most W x H (the centred fallback crop included), so kmax is at most that of the whole image.  Val: the box is a
  // function of (W, H), so the bound is exact; its filter may read outside the box (clamp = false), inside the image.
  size_t stage_bound(int W, int H) const {
    if (cfg_.train) return stage_bytes(W, H, cfg_.out_w, kmax_for(W, cfg_.out_w), cfg_.out_h, kmax_for(H, cfg_.out_h));
    Scratch s;
    return plan(s, W, H, center_crop(W, H, cfg_.out_w, cfg_.out_h, cfg_.resize_ratio)).bytes;
  }

  // test hook: bytes staged for sample `pos` of `epoch` if its record is W x H
  size_t stage_size(int64_t epoch, int64_t pos, int W, int H) const {
    Scratch s;
    return plan(s, W, H, box_for(uint64_t(epoch), uint64_t(pos), W, H)).bytes;
  }

 private:
  struct Plan { int x0, y0, rw, rh; size_t bytes; };

  Plan plan(Scratch& s, int W, int H, const Box& b) const {
    build_box_taps(s, W, H, b, cfg_.out_w, cfg_.out_h);
    const auto [x0, x1] = tap_span(s.tx);
    const auto [y0, y1] = tap_span(s.ty);
    return {x0, y0, x1 - x0, y1 - y0, stage_bytes(x1 - x0, y1 - y0, cfg_.out_w, s.tx.kmax, cfg_.out_h, s.ty.kmax)};
  }

  int rows_bound(int W, int H) const {
    if (cfg_.train) return kmax_for(H, cfg_.out_h);
    Scratch s;
    build_box_taps(s, W, H, center_crop(W, H, cfg_.out_w, cfg_.out_h, cfg_.resize_ratio), cfg_.out_w, cfg_.out_h);
    return s.ty.kmax;
  }

  // Copy the region and taps of sample i of the batch in `slot` into its arena and write its descriptor.
  void stage(const Record& r, const Box& b, int slot, size_t i, Scratch& s) {
    const Plan p = plan(s, int(r.w), int(r.h), b);
    const size_t table = table_bytes(cfg_.batch);
    const size_t off = stage_used_[slot].fetch_add(p.bytes);
    if (off + p.bytes > stage_cap_ - table) throw std::runtime_error("staging arena overflow (bound violated)");
    uint8_t* arena = reinterpret_cast<uint8_t*>(images_[slot]);
    uint8_t* region = arena + table + off;
    const size_t row = size_t(p.rw) * 3;
    for (int y = 0; y < p.rh; ++y)
      std::memcpy(region + y * row, r.px + (size_t(p.y0 + y) * r.w + p.x0) * 3, row);
    uint8_t* taps = region + align_up(row * p.rh);
    put_taps(put_taps(taps, s.tx, p.x0), s.ty, p.y0);
    StageDesc d{int64_t(region - arena), int64_t(taps - arena), p.rw, p.rh, s.tx.kmax, s.ty.kmax};
    std::memcpy(arena + i * sizeof(StageDesc), &d, sizeof d);
  }

  int batch_size_of(size_t k) const {
    const size_t begin = k * cfg_.batch;
    return int(std::min(size_t(cfg_.batch), per_rank_ - begin));
  }

  void build_order(uint64_t epoch) {
    const size_t n = records_.size();
    std::vector<uint32_t> perm(n);
    for (size_t i = 0; i < n; ++i) perm[i] = uint32_t(i);
    if (cfg_.shuffle) {                                  // Fisher-Yates, same stream on every rank
      Rng rng(mix(cfg_.seed, epoch, 0x5EED));
      for (size_t i = n - 1; i > 0; --i) std::swap(perm[i], perm[rng.below(i + 1)]);
    }
    order_.resize(per_rank_);
    for (size_t j = 0; j < per_rank_; ++j) order_[j] = perm[(j * cfg_.world + cfg_.rank) % n];
  }

  Box box_for(uint64_t epoch, uint64_t pos, int W, int H) const {
    if (!cfg_.train) return center_crop(W, H, cfg_.out_w, cfg_.out_h, cfg_.resize_ratio);
    Rng rng(mix(cfg_.seed, epoch, (pos * cfg_.world + cfg_.rank) * 2 + 1));
    Box b = random_resized_crop(rng, W, H, cfg_.scale_lo, cfg_.scale_hi, cfg_.ratio_lo, cfg_.ratio_hi);
    b.flip = rng.uniform() < 0.5;
    return b;
  }

  void work() {
    Scratch scratch;
    const size_t total = std::min(n_batches_ * size_t(cfg_.batch), per_rank_);
    const size_t img_bytes = size_t(3) * cfg_.out_h * cfg_.out_w;
    try {
      for (;;) {
        const size_t item = next_item_.fetch_add(1);
        if (item >= total) return;
        const size_t k = item / cfg_.batch, i = item % cfg_.batch;
        const int slot = int(k % cfg_.depth);
        {
          std::unique_lock<std::mutex> lk(mu_);          // wait until the consumer has released batch k - depth
          cv_free_.wait(lk, [&] { return quit_ || k < released_ + size_t(cfg_.depth); });
          if (quit_) return;
        }
        const uint32_t rec = order_[item];
        const Record& r = records_[rec];
        const Box b = box_for(epoch_, item, int(r.w), int(r.h));
        if (cfg_.staged) stage(r, b, slot, i, scratch);
        else resample(r, b, cfg_.out_w, cfg_.out_h, reinterpret_cast<uint8_t*>(images_[slot]) + i * img_bytes, scratch);
        reinterpret_cast<int64_t*>(labels_[slot])[i] = r.label;
        if (!ids_.empty()) reinterpret_cast<int64_t*>(ids_[slot])[i] = int64_t(rec);
        bool complete;
        {
          std::lock_guard<std::mutex> lk(mu_);
          complete = (++slot_done_[slot] == batch_size_of(k));
        }
        if (complete) cv_done_.notify_all();
      }
    } catch (const std::exception& e) {
      {
        std::lock_guard<std::mutex> lk(mu_);
        error_ = std::string("loader worker failed: ") + e.what();
      }
      cv_done_.notify_all();
    }
  }

  Config cfg_;
  std::vector<std::unique_ptr<Shard>> shards_;
  std::vector<Record> records_;
  size_t per_rank_ = 0, n_batches_ = 0;
  std::vector<uint32_t> order_;
  uint64_t epoch_ = 0;
  std::vector<uintptr_t> images_, labels_, ids_;

  std::vector<std::thread> workers_;
  std::atomic<size_t> next_item_{0};
  std::mutex mu_;
  std::condition_variable cv_done_, cv_free_;
  std::vector<int> slot_done_;
  std::unique_ptr<std::atomic<size_t>[]> stage_used_;      // per slot: bump pointer of the arena, after the descriptors
  size_t stage_cap_ = 0;
  int max_rows_ = 1;
  size_t consumed_ = 0, released_ = 0;
  bool quit_ = false;
  std::string error_;
};

// one-off resample entry for tests and tools: src HWC uint8 -> dst CHW uint8
void resample_once(uintptr_t src, int H, int W, double x0, double y0, double bw, double bh, bool clamp, bool flip, uintptr_t dst,
                   int out_h, int out_w) {
  Record r{reinterpret_cast<const uint8_t*>(src), uint32_t(H), uint32_t(W), 0};
  Box b{x0, y0, bw, bh, clamp, flip};
  Scratch s;
  resample(r, b, out_w, out_h, reinterpret_cast<uint8_t*>(dst), s);
}

}  // namespace

PYBIND11_MODULE(_L, m) {
  m.doc() = "native shard loader (host side of the input pipeline)";
  m.attr("INDEX_ENTRY_BYTES") = int(sizeof(IndexEntry));
  m.attr("MAGIC") = py::bytes(kMagic, 8);
  py::class_<ShardLoader>(m, "ShardLoader")
      .def(py::init([](const std::vector<std::string>& paths, int batch, int out_h, int out_w, bool train, uint64_t seed, int rank,
                       int world, int threads, int depth, bool drop_last, bool shuffle, double scale_lo, double scale_hi,
                       double ratio_lo, double ratio_hi, double resize_ratio, bool staged) {
             Config c{batch, out_h, out_w, train, seed, rank, world, threads, depth, drop_last, shuffle,
                      scale_lo, scale_hi, ratio_lo, ratio_hi, resize_ratio, staged};
             return new ShardLoader(paths, c);
           }),
           py::arg("paths"), py::arg("batch"), py::arg("out_h"), py::arg("out_w"), py::arg("train"), py::arg("seed"), py::arg("rank"),
           py::arg("world"), py::arg("threads"), py::arg("depth"), py::arg("drop_last"), py::arg("shuffle"),
           py::arg("scale_lo") = 0.08, py::arg("scale_hi") = 1.0, py::arg("ratio_lo") = 0.75, py::arg("ratio_hi") = 4.0 / 3.0,
           py::arg("resize_ratio") = 256.0 / 224.0, py::arg("staged") = false)
      .def("size", &ShardLoader::size)
      .def("samples_per_rank", &ShardLoader::samples_per_rank)
      .def("num_batches", &ShardLoader::num_batches)
      .def("depth", &ShardLoader::depth)
      .def("set_buffers", &ShardLoader::set_buffers, py::arg("images"), py::arg("labels"), py::arg("ids") = std::vector<uintptr_t>())
      .def("start_epoch", &ShardLoader::start_epoch, py::call_guard<py::gil_scoped_release>())
      .def("next", &ShardLoader::next, py::call_guard<py::gil_scoped_release>())
      .def("release", &ShardLoader::release)
      .def("stop", &ShardLoader::stop, py::call_guard<py::gil_scoped_release>())
      .def("crop_params", &ShardLoader::crop_params)
      .def("epoch_order", &ShardLoader::epoch_order)
      .def("stage_capacity", &ShardLoader::stage_capacity)
      .def("stage_max_rows", &ShardLoader::stage_max_rows)
      .def("staged_bytes", &ShardLoader::staged_bytes)
      .def("stage_bound", &ShardLoader::stage_bound)
      .def("stage_size", &ShardLoader::stage_size);
  m.attr("STAGE_DESC_BYTES") = int(sizeof(StageDesc));
  m.def("resample", &resample_once, py::call_guard<py::gil_scoped_release>());
}
