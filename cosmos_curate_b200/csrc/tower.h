// Host-side parts the transformer tower handles (cb_vit, cb_iv2, cb_iv2_text) share: the weight store each declares its tensors in,
// the workspace of device buffers sized at finalize, and the loop that runs a call in chunks of that workspace.
#pragma once
#include <cuda_fp16.h>

#include <algorithm>
#include <cassert>
#include <string>
#include <vector>

#include "common.h"

namespace cb {

enum Storage { F32, F16 };  // F16: GEMM weights, converted from the fp32 input with round-to-nearest-even

// The tensors a tower accepts, indexed by the tower's enums: the tensors outside the layers are 0 .. globals - 1, and leaf j of layer i
// (named "L<i>.<leaf>") is globals + i * leaves + j.  An entry left unnamed is not part of the tower's configuration.
class WeightStore {
 public:
  WeightStore() = default;
  WeightStore(const WeightStore&) = delete;
  WeightStore& operator=(const WeightStore&) = delete;
  ~WeightStore() {
    for (Tensor& x : t_) cudaFree(x.d);
  }

  void layout(int globals, int leaves, int layers) {
    globals_ = globals, leaves_ = leaves, layers_ = layers;
    t_.resize(globals + (size_t)leaves * layers);
  }
  // cols > 0: rows of `cols` values are stored zero-padded to `pad_cols` (patch_w: 3 * patch^2 -> k_pad)
  void add(int id, std::string name, size_t count, Storage s = F32, size_t cols = 0, size_t pad_cols = 0) {
    t_[id] = {std::move(name), count, s, cols, pad_cols};
  }
  void add_leaf(int leaf, const char* name, size_t count, Storage s = F32) {
    for (int i = 0; i < layers_; ++i) add(globals_ + i * leaves_ + leaf, "L" + std::to_string(i) + "." + name, count, s);
  }

  // Validates `name` and `count` against the table and uploads the tensor; `who` prefixes the messages ("vit" -> "vit_set_tensor: ...").
  int set(cb_ctx* ctx, const char* who, const char* name, const float* data, size_t count) {
    if (!name || !data) return fail(ctx, CB_ERR_ARG, "%s_set_tensor: null argument", who);
    auto it = std::find_if(t_.begin(), t_.end(), [&](const Tensor& x) { return !x.name.empty() && x.name == name; });
    if (it == t_.end()) return fail(ctx, CB_ERR_ARG, "%s_set_tensor: unknown tensor '%s'", who, name);
    Tensor& x = *it;
    if (x.count != count) return fail(ctx, CB_ERR_ARG, "%s_set_tensor: '%s' has %zu elements, expected %zu", who, name, count, x.count);
    cudaFree(x.d), x.d = nullptr;
    const void* src = data;
    size_t bytes = count * sizeof(float);
    std::vector<__half> hbuf;
    if (x.storage == F16) {
      const size_t cols = x.cols ? x.cols : count, out_cols = x.cols ? x.pad_cols : count, rows = count / cols;
      hbuf.assign(rows * out_cols, __float2half_rn(0.f));
      for (size_t r = 0; r < rows; ++r)
        for (size_t c = 0; c < cols; ++c) hbuf[r * out_cols + c] = __float2half_rn(data[r * cols + c]);
      src = hbuf.data(), bytes = hbuf.size() * sizeof(__half);
    }
    CB_CUDA(ctx, cudaMalloc(&x.d, bytes));
    CB_CUDA(ctx, cudaMemcpy(x.d, src, bytes, cudaMemcpyHostToDevice));
    return CB_OK;
  }

  // `who`: "vit_finalize" -> "vit_finalize: tensor '...' was never set"
  int check_complete(cb_ctx* ctx, const char* who) const {
    for (const Tensor& x : t_)
      if (!x.name.empty() && !x.d) return fail(ctx, CB_ERR_STATE, "%s: tensor '%s' was never set", who, x.name.c_str());
    return CB_OK;
  }

  // Device pointers for the forward, valid after a successful check_complete; asking for a tensor outside the configuration, or of the
  // other storage, is a schedule bug.
  const float* f(int id) const { return (const float*)get(id, F32); }
  const void* h(int id) const { return get(id, F16); }
  const float* f(int layer, int leaf) const { return f(globals_ + layer * leaves_ + leaf); }
  const void* h(int layer, int leaf) const { return h(globals_ + layer * leaves_ + leaf); }

 private:
  struct Tensor {
    std::string name;
    size_t count = 0;
    Storage storage = F32;
    size_t cols = 0, pad_cols = 0;
    void* d = nullptr;
  };
  const void* get(int id, Storage s) const {
    assert(t_[id].d && t_[id].storage == s);
    return t_[id].d;
  }
  std::vector<Tensor> t_;
  int globals_ = 0, leaves_ = 0, layers_ = 0;
};

// A handle's device buffers: one cudaMalloc each, because their addresses and alignment feed the GEMM's TMA descriptors.
class Workspace {
 public:
  Workspace() = default;
  Workspace(const Workspace&) = delete;
  Workspace& operator=(const Workspace&) = delete;
  ~Workspace() { release(); }

  template <typename T>
  int alloc(cb_ctx* ctx, T** p, size_t count) {
    CB_CUDA(ctx, cudaMalloc((void**)p, count * sizeof(T)));
    bufs_.push_back((void**)p);
    return CB_OK;
  }
  // Frees every buffer alloc recorded and nulls its pointer.
  void release() {
    for (void** p : bufs_) cudaFree(*p), *p = nullptr;
    bufs_.clear();
  }

 private:
  std::vector<void**> bufs_;
};

// fn(first, count) over [0, n) in chunks of at most `cap` items; stops at the first error.
template <typename Fn>
int for_chunks(int n, int cap, Fn&& fn) {
  for (int i = 0; i < n; i += cap)
    if (const int rc = fn(i, std::min(cap, n - i))) return rc;
  return CB_OK;
}

}  // namespace cb
