// NCCL communicator wrappers (multi-GPU landmark sharding: one sum-allreduce of the reduced camera
// system per LM step over NVLink / NVSwitch).
//
// NCCL is bound at run time (dlopen) the first time a communicator is requested, not at link time:
//  * single-GPU users do not need NCCL at all;
//  * a host process that also loads another NCCL user (e.g. PyTorch ships its own libnccl.so.2, newer
//    than the system one) ends up with ONE copy: dlopen by soname returns whichever is already mapped.
// Lookup order: $CTVIO_NCCL_LIB, then "libnccl.so.2", then "libnccl.so".
#include <dlfcn.h>
#include <nccl.h>  // types and enums only; no symbol from it is linked

#include <cstdlib>
#include <mutex>

#include "marginalize.h"

namespace ctvio {

static_assert(sizeof(ncclUniqueId) == 128, "ctvio_nccl_unique_id hands out 128 bytes");

namespace {

struct NcclApi {
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  std::string load_error;
  bool ok = false;
};

NcclApi& nccl_api() {
  static NcclApi api;
  static std::once_flag once;
  std::call_once(once, [] {
    void* h = nullptr;
    const char* env = std::getenv("CTVIO_NCCL_LIB");
    const char* names[3] = {env, "libnccl.so.2", "libnccl.so"};
    for (const char* nm : names) {
      if (!nm || !*nm) continue;
      h = dlopen(nm, RTLD_NOW | RTLD_GLOBAL);
      if (h) break;
    }
    if (!h) {
      const char* e = dlerror();
      api.load_error = std::string("cannot load NCCL (set CTVIO_NCCL_LIB): ") + (e ? e : "unknown");
      return;
    }
    auto sym = [&](const char* nm) -> void* {
      void* p = dlsym(h, nm);
      if (!p && api.load_error.empty()) api.load_error = std::string("NCCL symbol missing: ") + nm;
      return p;
    };
    api.GetUniqueId = reinterpret_cast<decltype(api.GetUniqueId)>(sym("ncclGetUniqueId"));
    api.CommInitRank = reinterpret_cast<decltype(api.CommInitRank)>(sym("ncclCommInitRank"));
    api.CommDestroy = reinterpret_cast<decltype(api.CommDestroy)>(sym("ncclCommDestroy"));
    api.AllReduce = reinterpret_cast<decltype(api.AllReduce)>(sym("ncclAllReduce"));
    api.AllGather = reinterpret_cast<decltype(api.AllGather)>(sym("ncclAllGather"));
    api.GetErrorString = reinterpret_cast<decltype(api.GetErrorString)>(sym("ncclGetErrorString"));
    api.ok = api.load_error.empty();
  });
  return api;
}

bool fail(std::string* err, const char* what, ncclResult_t r) {
  if (err) *err = std::string(what) + ": " + nccl_api().GetErrorString(r);
  return false;
}

}  // namespace

bool comm_unique_id(uint8_t* id128, std::string* err) {
  NcclApi& n = nccl_api();
  if (!n.ok) {
    if (err) *err = n.load_error;
    return false;
  }
  ncclUniqueId id;
  ncclResult_t r = n.GetUniqueId(&id);
  if (r != ncclSuccess) return fail(err, "ncclGetUniqueId", r);
  memcpy(id128, &id, 128);
  return true;
}

void* comm_create(int rank, int world, const uint8_t* id128, std::string* err) {
  NcclApi& n = nccl_api();
  if (!n.ok) {
    if (err) *err = n.load_error;
    return nullptr;
  }
  ncclUniqueId id;
  memcpy(&id, id128, 128);
  ncclComm_t comm = nullptr;
  ncclResult_t r = n.CommInitRank(&comm, world, id, rank);
  if (r != ncclSuccess) {
    fail(err, "ncclCommInitRank", r);
    return nullptr;
  }
  return comm;
}

void comm_destroy(void* comm) {
  if (comm && nccl_api().ok) nccl_api().CommDestroy(static_cast<ncclComm_t>(comm));
}

bool comm_allreduce_sum(void* comm, double* buf, size_t n, cudaStream_t s, std::string* err) {
  ncclResult_t r = nccl_api().AllReduce(buf, buf, n, ncclDouble, ncclSum, static_cast<ncclComm_t>(comm), s);
  if (r != ncclSuccess) return fail(err, "ncclAllReduce", r);
  return true;
}

bool comm_allgather(void* comm, const double* send, double* recv, size_t n_per_rank, cudaStream_t s, std::string* err) {
  ncclResult_t r = nccl_api().AllGather(send, recv, n_per_rank, ncclDouble, static_cast<ncclComm_t>(comm), s);
  if (r != ncclSuccess) return fail(err, "ncclAllGather", r);
  return true;
}

}  // namespace ctvio
