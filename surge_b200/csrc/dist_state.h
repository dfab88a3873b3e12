// dist_state.h — state of one rank of the multi-GPU replay (shared by dist.cu and route_push.cu).
#pragma once
#include <cuda_runtime.h>
#include <nccl.h>
#include <stdint.h>

#include <condition_variable>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "devbuf.h"
#include "dist.cuh"

namespace sgr {

// Every rank's receive allocation starts with a header the other ranks write arrival flags into
// (u64 flags[kMaxRanks][kMaxChunks]: (epoch << 32) | records + 1 of region (source, chunk)); the records follow.
constexpr size_t kRecvHeaderBytes = 64 << 10;
constexpr int kMaxChunks = 256;

struct NcclApi {
  void* lib = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  ncclResult_t (*Send)(const void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Recv)(void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  bool load(std::string* err);
};
NcclApi& nccl_api();

// The exchange code's error path: a failed CUDA (DTRY) or NCCL (NTRY) call puts its source text and the library's reason into
// *err and returns SGR_ERR_CUDA / SGR_ERR_DIST. DTRY needs `cudaError_t ce` and both need `std::string* err` in scope.
#define DTRY(x) if ((ce = (x)) != cudaSuccess) { *err = std::string(#x ": ") + cudaGetErrorString(ce); return SGR_ERR_CUDA; }
#define NTRY(x) { ncclResult_t _r = (x); if (_r != ncclSuccess) { *err = std::string(#x ": ") + nccl_api().GetErrorString(_r); return SGR_ERR_DIST; } }

// Loopback ranks are streams of one process on one device, and streams share the device's hardware queues, each run in order.
// A fold launch that waits for its rank's spinning wait kernel can stand at the head of a queue and hold back a peer's partition
// or flag kernel queued behind it, and the wait spins until its limit. So every loopback rank enqueues all its partition and flag
// kernels, meets its peers here, and only then enqueues its waits and folds: nothing a wait needs is ever queued behind a wait.
struct LoopbackGroup {
  std::mutex mu;
  std::condition_variable cv;
  int nranks = 0, arrived = 0;
  uint64_t generation = 0;
  bool arrive_and_wait(int seconds);   // false: a peer did not arrive in time (it left the barrier as it found it)
};

struct DistState {
  int rank = 0, nranks = 1;
  bool loopback = false;                 // several ranks inside one process (tests): no NCCL, peers handed over as raw pointers
  ncclComm_t comm = nullptr;
  uint64_t n_global = 0, n_local = 0;
  DevBuf owner_of, local_of, global_of_local, part_tmp, flags, pos, scan_tmp;
  DevBuf hist, owner_total, counts_all, send_buf, recv_buf;
  uint64_t recv_capacity = 0;            // records
  uint8_t* peer_recv[kMaxRanks] = {};    // every rank's receive RECORDS (behind the header), mapped here
  uint8_t* peer_base[kMaxRanks] = {};    // every rank's receive allocation (header first)
  bool peers_mapped = false;
  std::vector<void*> opened;             // IPC mappings to close
  DistStats stats{};
  Event ev[6];
  // pipelined push path (route_push.cu)
  DevBuf route_of;                       // owner << 28 | local index, per global aggregate
  DevBuf lb, push_ctl, gather_buf;       // look-back cells; tickets + chunk totals + status; contiguous copy for the replay
  Stream stream2, stream_hi;             // fold (low priority) and partition (high priority) streams
  Event pev[4];
  uint32_t epoch = 0;
  HostBuf h_pinned;                      // page-locked landing area of the per-call read-backs
  std::shared_ptr<LoopbackGroup> group;  // loopback ranks: shared by the ranks whose rank 0 has the same receive allocation

  // Closes the peers' IPC mappings and the NCCL communicator; the members then free what this rank allocated.
  ~DistState();
};

}  // namespace sgr
