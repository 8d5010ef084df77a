/*
 * teb_comm.h — the one collective of the path: all-gather of the per-candidate costs over NCCL (NVLink / NVSwitch).
 *
 * The reference fans the candidates of one planning cycle out to threads and picks the best one afterwards
 * (homotopy_class_planner.cpp:466-493 optimizeAllTEBs, :564-616 selectBestTeb). With one process per GPU the batch axis
 * is sharded, bands never exchange anything while they are optimised, and selection needs exactly the costs of all
 * shards: one ncclAllGather of count_local doubles per rank on the context's stream (<= 64 KB, latency bound).
 *
 * NCCL is resolved at run time (dlopen of libnccl.so.2, i.e. the copy the process already loaded - torch's - or the
 * system one): libteb_b200.so has no link-time dependency on it and single-GPU users never load it.
 */
#pragma once
#include <dlfcn.h>
#include <nccl.h>

#include <mutex>
#include <string>

namespace tebgpu {

struct NcclApi {
  void* handle = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  ncclResult_t (*GetVersion)(int*) = nullptr;
  std::string error;
  bool ok() const { return handle != nullptr && error.empty(); }
};

inline NcclApi& nccl_api() {
  static NcclApi api;
  static std::once_flag once;
  std::call_once(once, [] {
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char* nm : names) {
      api.handle = dlopen(nm, RTLD_NOW | RTLD_GLOBAL);
      if (api.handle) break;
    }
    if (!api.handle) { api.error = std::string("dlopen(libnccl.so.2) failed: ") + (dlerror() ? dlerror() : "?"); return; }
    auto sym = [&](const char* s) -> void* {
      void* p = dlsym(api.handle, s);
      if (!p && api.error.empty()) api.error = std::string("NCCL symbol missing: ") + s;
      return p;
    };
    api.GetUniqueId = reinterpret_cast<decltype(api.GetUniqueId)>(sym("ncclGetUniqueId"));
    api.CommInitRank = reinterpret_cast<decltype(api.CommInitRank)>(sym("ncclCommInitRank"));
    api.CommDestroy = reinterpret_cast<decltype(api.CommDestroy)>(sym("ncclCommDestroy"));
    api.AllGather = reinterpret_cast<decltype(api.AllGather)>(sym("ncclAllGather"));
    api.GroupStart = reinterpret_cast<decltype(api.GroupStart)>(sym("ncclGroupStart"));
    api.GroupEnd = reinterpret_cast<decltype(api.GroupEnd)>(sym("ncclGroupEnd"));
    api.GetErrorString = reinterpret_cast<decltype(api.GetErrorString)>(sym("ncclGetErrorString"));
    api.GetVersion = reinterpret_cast<decltype(api.GetVersion)>(sym("ncclGetVersion"));
  });
  return api;
}

}  // namespace tebgpu
