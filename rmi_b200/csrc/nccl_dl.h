// nccl_dl.h — NCCL bound at run time (dlopen), so that librmi_b200.so has no link-time dependency
// on it: single-GPU users never load NCCL, and inside a torch process the already-loaded
// libnccl.so.2 (the one torch.distributed uses) is the one that gets picked up.
//
// Only the handful of entry points the range-partitioned build and lookups issue are bound; types and
// enumerators come from the system header (ABI-stable across the 2.x series).
#pragma once
#include <dlfcn.h>
#include <nccl.h>

#include <mutex>
#include <string>

namespace rmi {

struct NcclApi {
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Broadcast)(const void*, void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Send)(const void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Recv)(void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  ncclResult_t (*GetVersion)(int*) = nullptr;
  std::string error;   // why loading failed ("" = loaded)
  bool ok = false;
};

inline const NcclApi& nccl_api() {
  static NcclApi api;
  static std::once_flag once;
  std::call_once(once, [] {
    void* h = nullptr;
    for (const char* name : {"libnccl.so.2", "libnccl.so"}) {
      h = dlopen(name, RTLD_NOW | RTLD_GLOBAL);
      if (h) break;
    }
    if (!h) { api.error = std::string("dlopen(libnccl.so.2) failed: ") + dlerror(); return; }
    auto bind = [&](auto& fn, const char* sym) {
      fn = reinterpret_cast<std::remove_reference_t<decltype(fn)>>(dlsym(h, sym));
      if (!fn && api.error.empty()) api.error = std::string("NCCL symbol not found: ") + sym;
    };
    bind(api.GetUniqueId, "ncclGetUniqueId");
    bind(api.CommInitRank, "ncclCommInitRank");
    bind(api.CommDestroy, "ncclCommDestroy");
    bind(api.GetErrorString, "ncclGetErrorString");
    bind(api.AllReduce, "ncclAllReduce");
    bind(api.AllGather, "ncclAllGather");
    bind(api.Broadcast, "ncclBroadcast");
    bind(api.Send, "ncclSend");
    bind(api.Recv, "ncclRecv");
    bind(api.GroupStart, "ncclGroupStart");
    bind(api.GroupEnd, "ncclGroupEnd");
    bind(api.GetVersion, "ncclGetVersion");
    api.ok = api.error.empty();
  });
  return api;
}

}  // namespace rmi
