// mloam_context.hpp — one GPU context per host thread + error mapping, shared by mloam_shim.hpp (POD stand-in types) and
// mloam_adapter.hpp (the reference's own PCL / Eigen / Ceres types).
#pragma once
#include <stdexcept>
#include <string>

#include "../../include/mloam_b200.h"

namespace mloam {

inline void check(mloam_ctx_t *ctx, int rc, const char *what) {
  if (rc != MLOAM_OK) throw std::runtime_error(std::string(what) + ": " + (ctx ? mloam_last_error(ctx) : "no context"));
}

// One context per host thread (the reference's objects are shared between OpenMP threads, the GPU state is not).
class ThreadContext {
 public:
  static mloam_ctx_t *get(int device = 0) {
    thread_local ThreadContext tc(device);
    return tc.ctx_;
  }
  static mloam_params_t &params() {
    static mloam_params_t p = [] {
      mloam_params_t q;
      mloam_default_params(&q);
      return q;
    }();
    return p;
  }
  // Push the (mutable, global — like the reference's parameters.h globals) parameters to this thread's context.
  static void applyParams() { check(get(), mloam_set_params(get(), &params()), "mloam_set_params"); }

 private:
  explicit ThreadContext(int device) {
    if (mloam_ctx_create(device, &params(), &ctx_) != MLOAM_OK)
      throw std::runtime_error("mloam_ctx_create failed: an H100 (sm_90a) device is required — there is no CPU path");
  }
  ~ThreadContext() { mloam_ctx_destroy(ctx_); }
  mloam_ctx_t *ctx_ = nullptr;
};

}  // namespace mloam
