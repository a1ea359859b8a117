// comm.cu — multi-GPU plumbing: one LiDAR per GPU, one all-reduce of the packed normal equations per LM
// evaluation (SURVEY.md §8e).  NCCL over NVLink / NVSwitch; the collective is enqueued on the context stream
// between the block-partial reduction and the LM step, so an iteration never returns to the host.
#include <dlfcn.h>
#include <nccl.h>  // types and prototypes only: the library is bound at run time (see nccl_api())

#include <cstring>

#include "ctx.h"
#include "host_util.h"

using namespace mloam;

// NCCL is resolved with dlopen instead of a link-time dependency: a process that also hosts PyTorch already
// carries torch's bundled libnccl.so.2, and binding a second copy at load time would clash with it.  dlopen
// returns the resident library when there is one, the system library otherwise.
namespace {
struct NcclApi {
  decltype(&ncclGetUniqueId) GetUniqueId = nullptr;
  decltype(&ncclCommInitRank) CommInitRank = nullptr;
  decltype(&ncclAllReduce) AllReduce = nullptr;
  decltype(&ncclCommDestroy) CommDestroy = nullptr;
  decltype(&ncclGetErrorString) GetErrorString = nullptr;
  bool ok = false;
};
NcclApi *nccl_api() {
  static NcclApi api;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void *h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);
    if (!h) h = dlopen("libnccl.so.2", RTLD_NOW);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW);
    if (h) {
      api.GetUniqueId = (decltype(api.GetUniqueId))dlsym(h, "ncclGetUniqueId");
      api.CommInitRank = (decltype(api.CommInitRank))dlsym(h, "ncclCommInitRank");
      api.AllReduce = (decltype(api.AllReduce))dlsym(h, "ncclAllReduce");
      api.CommDestroy = (decltype(api.CommDestroy))dlsym(h, "ncclCommDestroy");
      api.GetErrorString = (decltype(api.GetErrorString))dlsym(h, "ncclGetErrorString");
      api.ok = api.GetUniqueId && api.CommInitRank && api.AllReduce && api.CommDestroy && api.GetErrorString;
    }
  }
  return api.ok ? &api : nullptr;
}
}  // namespace

namespace mloam {
int comm_allreduce_doubles(Ctx *c, double *d_buf, int count) {
  if (!c->nccl_comm) return MLOAM_OK;
  ncclResult_t r = nccl_api()->AllReduce(d_buf, d_buf, (size_t)count, ncclDouble, ncclSum, (ncclComm_t)c->nccl_comm, c->stream);
  if (r != ncclSuccess) {
    c->err = std::string("ncclAllReduce: ") + nccl_api()->GetErrorString(r);
    return MLOAM_E_NCCL;
  }
  return MLOAM_OK;
}
}  // namespace mloam

extern "C" {

int mloam_comm_unique_id(void *id128) {
  if (!id128) return MLOAM_E_INVALID;
  static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
  ncclUniqueId id;
  if (!nccl_api() || nccl_api()->GetUniqueId(&id) != ncclSuccess) return MLOAM_E_NCCL;
  memcpy(id128, &id, sizeof(id));
  return MLOAM_OK;
}

int mloam_comm_init(mloam_ctx_t *h, int nranks, int rank, const void *id128) {
  if (!h || !id128 || nranks < 1 || rank < 0 || rank >= nranks) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  cudaSetDevice(c->device);
  if (c->nccl_comm) mloam_comm_destroy(h);
  ncclUniqueId id;
  memcpy(&id, id128, sizeof(id));
  ncclComm_t comm;
  if (!nccl_api()) return fail(c, MLOAM_E_NCCL, "libnccl.so.2 could not be loaded");
  ncclResult_t r = nccl_api()->CommInitRank(&comm, nranks, id, rank);
  if (r != ncclSuccess) {
    c->err = std::string("ncclCommInitRank: ") + nccl_api()->GetErrorString(r);
    return MLOAM_E_NCCL;
  }
  c->nccl_comm = comm;
  c->nranks = nranks, c->rank = rank;
  return MLOAM_OK;
}

// ---- peer-memory exchange (replaces the NCCL all-reduce on the LM path when every GPU can map every other)
int mloam_comm_p2p_export(mloam_ctx_t *h, void *handle64) {
  if (!h || !handle64) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  cudaSetDevice(c->device);
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
  if (!c->p2p_local) {
    MLOAM_CUDA_OK(c, cudaMalloc(&c->p2p_local, MLOAM_P2P_BYTES));
    MLOAM_CUDA_OK(c, cudaMemset(c->p2p_local, 0, MLOAM_P2P_BYTES));
    MLOAM_CUDA_OK(c, cudaDeviceSynchronize());
  }
  cudaIpcMemHandle_t hd;
  MLOAM_CUDA_OK(c, cudaIpcGetMemHandle(&hd, c->p2p_local));
  memcpy(handle64, &hd, sizeof(hd));
  return MLOAM_OK;
}

int mloam_comm_p2p_init(mloam_ctx_t *h, int nranks, int rank, const void *handles) {
  if (!h || !handles || nranks < 2 || nranks > MLOAM_P2P_MAX_RANKS || rank < 0 || rank >= nranks) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  cudaSetDevice(c->device);
  if (!c->p2p_local) return fail(c, MLOAM_E_STATE, "comm_p2p_init: call mloam_comm_p2p_export first");
  for (int q = 0; q < nranks; q++) {
    if (q == rank) {
      c->p2p_peer[q] = c->p2p_local;
      continue;
    }
    cudaIpcMemHandle_t hd;
    memcpy(&hd, static_cast<const char *>(handles) + 64 * (size_t)q, sizeof(hd));
    void *ptr = nullptr;
    cudaError_t e = cudaIpcOpenMemHandle(&ptr, hd, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) {
      cudaGetLastError();
      for (int k = 0; k < q; k++)
        if (k != rank && c->p2p_peer[k]) cudaIpcCloseMemHandle(c->p2p_peer[k]), c->p2p_peer[k] = nullptr;
      c->err = std::string("cudaIpcOpenMemHandle: ") + cudaGetErrorString(e);
      return MLOAM_E_CUDA;
    }
    c->p2p_peer[q] = ptr;
  }
  c->nranks = nranks, c->rank = rank;
  P2PView v;
  memset(&v, 0, sizeof(v));
  for (int q = 0; q < nranks; q++) {
    char *base = static_cast<char *>(c->p2p_peer[q]);
    v.flags[q] = reinterpret_cast<unsigned *>(base + 64), v.slots[q] = reinterpret_cast<double *>(base + 256);
  }
  v.epoch = reinterpret_cast<unsigned long long *>(c->p2p_local);
  v.nranks = nranks, v.rank = rank;
  if (!c->p2p_view) MLOAM_CUDA_OK(c, cudaMalloc(&c->p2p_view, sizeof(P2PView)));
  MLOAM_CUDA_OK(c, cudaMemcpy(c->p2p_view, &v, sizeof(v), cudaMemcpyHostToDevice));
  c->p2p_on = true;
  return MLOAM_OK;
}

// Re-synchronise after a failed exchange (termination 9): every rank calls this BETWEEN two host barriers (no rank may be inside
// a collective solve); flags, slots and the epoch of the local buffer go back to zero, so all ranks restart at exchange 0.
int mloam_comm_p2p_reset(mloam_ctx_t *h) {
  if (!h) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  cudaSetDevice(c->device);
  if (!c->p2p_local) return MLOAM_OK;
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(c->stream));
  MLOAM_CUDA_OK(c, cudaMemset(c->p2p_local, 0, MLOAM_P2P_BYTES));
  MLOAM_CUDA_OK(c, cudaDeviceSynchronize());
  return MLOAM_OK;
}

int mloam_comm_destroy(mloam_ctx_t *h) {
  if (!h) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  if (c->p2p_local) {
    cudaStreamSynchronize(c->stream);
    for (int q = 0; q < MLOAM_P2P_MAX_RANKS; q++) {
      if (c->p2p_peer[q] && c->p2p_peer[q] != c->p2p_local) cudaIpcCloseMemHandle(c->p2p_peer[q]);
      c->p2p_peer[q] = nullptr;
    }
    cudaFree(c->p2p_local);
    c->p2p_local = nullptr;
    if (c->p2p_view) cudaFree(c->p2p_view), c->p2p_view = nullptr;
    c->p2p_on = false;
    if (!c->nccl_comm) c->nranks = 1, c->rank = 0;
  }
  if (c->nccl_comm) {
    cudaStreamSynchronize(c->stream);
    nccl_api()->CommDestroy((ncclComm_t)c->nccl_comm);
    c->nccl_comm = nullptr;
    c->nranks = 1, c->rank = 0;
  }
  return MLOAM_OK;
}

}  // extern "C"
