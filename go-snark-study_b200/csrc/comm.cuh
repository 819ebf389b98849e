// Multi-GPU plumbing INSIDE the library: one process per GPU, an NCCL communicator owned by libb200snark, so that a
// caller of the reference-facing entry point (groth16.GenerateProofs -> b200_groth16_prove) can use a sharded proving
// key with plain host pointers — the all-gather of the per-rank partial sums happens under the C ABI.
//
// The exchange step of the path (SURVEY §8e): every rank leaves a 1 KB record of partial sums (XYZZ: A | B1 | B2 | C+H
// with s*A_part + r*B1_part already folded into the C part); NCCL has no elliptic-curve reduction, so the records are
// all-gathered (1 KB per rank over NVLink / NVSwitch — latency only) and every rank adds them.
//
// libnccl is resolved at run time (dlopen) so the library has no link-time dependency and shares the copy a host
// process may already have loaded (a torch process: the torch-bundled libnccl.so.2).  Only the stable core API is used.
#pragma once
#include <dlfcn.h>
#include <nccl.h>

namespace b200 {

struct NcclApi {
  void* so = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*CommSplit)(ncclComm_t, int, int, ncclComm_t*, ncclConfig_t*) = nullptr;   // optional (NCCL >= 2.18)
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  const char* load() {
    if (so) return nullptr;
    for (const char* name : {"libnccl.so.2", "libnccl.so"}) {
      so = dlopen(name, RTLD_NOW | RTLD_GLOBAL);
      if (so) break;
    }
    if (!so) return "libnccl.so.2 not found (dlopen)";
    GetUniqueId = reinterpret_cast<decltype(GetUniqueId)>(dlsym(so, "ncclGetUniqueId"));
    CommInitRank = reinterpret_cast<decltype(CommInitRank)>(dlsym(so, "ncclCommInitRank"));
    CommDestroy = reinterpret_cast<decltype(CommDestroy)>(dlsym(so, "ncclCommDestroy"));
    AllGather = reinterpret_cast<decltype(AllGather)>(dlsym(so, "ncclAllGather"));
    GetErrorString = reinterpret_cast<decltype(GetErrorString)>(dlsym(so, "ncclGetErrorString"));
    CommSplit = reinterpret_cast<decltype(CommSplit)>(dlsym(so, "ncclCommSplit"));
    if (!GetUniqueId || !CommInitRank || !CommDestroy || !AllGather || !GetErrorString) {
      so = nullptr;
      return "libnccl: missing symbols";
    }
    return nullptr;
  }
};

// The communicators themselves belong to the prove contexts (capi.cu: ProveCtx).
struct Comm {
  NcclApi api;
  int rank = 0, world = 1;
};

static_assert(sizeof(ncclUniqueId) == 128, "b200_comm_unique_id hands out 128 bytes");

}  // namespace b200
