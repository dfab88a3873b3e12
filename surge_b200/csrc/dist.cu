// dist.cu — multi-GPU replay: route events to the rank that owns their aggregate, then group + fold.
//
// The reference shards by key: aggregateId -> Kafka partition (KafkaPartitionProvider.partitionForKey,
// modules/common/src/main/scala/surge/kafka/KafkaPartitioner.scala:7-9) -> consumer-group assignment -> node,
// with the BROKER doing the shuffle (KafkaProducerHelperCommon.getPartitionFor,
// modules/common/src/main/scala/surge/kafka/KafkaProducer.scala:45-57). Here one process per GPU holds the
// records of its source partitions in arrival order and the shuffle is ONE exchange over NVLink:
//
//   K4 route_count    owner histogram per 2048-record block                     (reads 8 B of every record)
//   exchange counts   nranks x nranks matrix (ncclAllGather, 8*nranks bytes per rank)
//   K4 route_scatter  stable partition by owner; every 64-byte record is written ONCE, straight to its
//                     destination: either this rank's send region (NCCL path) or the owner's receive
//                     buffer through a peer-mapped pointer (fused path: route + all-to-all in one kernel,
//                     coalesced 64-byte stores over NVLink, no staging copy)
//   exchange records  NCCL path only: grouped ncclSend/ncclRecv (one all-to-all)
//   K5 + fold         stable group-by of the received records by local aggregate index, then the fold
//
// Per-aggregate order survives because all events of an aggregate come from one source partition
// (one key -> one partition), both partition steps are stable, and the receiver keeps each source's
// block contiguous.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <nccl.h>
#include <stdio.h>
#include <string.h>

#include <chrono>
#include <map>
#include <string>
#include <vector>

#include "../../include/sgr.h"
#include "devbuf.h"
#include "dist.cuh"
#include "dist_state.h"
#include "group_kernels.cuh"

namespace sgr {
namespace {

constexpr int kRouteThreads = 256;
constexpr int kRouteBlockRecs = 2048;  // records per block (8 rounds of 256)

// ---------------------------------------------------------------- owner / local index tables
__global__ void owner_table_kernel(const uint32_t* __restrict__ partition_of, uint64_t n, uint32_t nranks,
                                   uint8_t* __restrict__ owner_of) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) owner_of[i] = (uint8_t)(partition_of[i] % nranks);
}
__global__ void owner_flags_kernel(const uint8_t* __restrict__ owner_of, uint64_t n, uint32_t r, uint32_t* __restrict__ flags) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) flags[i] = owner_of[i] == r ? 1u : 0u;
}
__global__ void local_index_kernel(const uint8_t* __restrict__ owner_of, uint64_t n, uint32_t r, const uint32_t* __restrict__ pos,
                                   uint32_t* __restrict__ local_of, uint32_t* __restrict__ global_of_local, uint32_t my_rank) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && owner_of[i] == r) {
    local_of[i] = pos[i];
    if (r == my_rank && global_of_local) global_of_local[pos[i]] = (uint32_t)i;
  }
}

__global__ void route_table_kernel(const uint8_t* __restrict__ owner_of, const uint32_t* __restrict__ local_of, uint64_t n, uint32_t* __restrict__ route_of) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) route_of[i] = ((uint32_t)owner_of[i] << 28) | (local_of[i] & 0x0fffffffu);
}

// my row of the count matrix: records per owner, my receive capacity, how many of my records carry a bad aggregate index
__global__ void route_row_kernel(const uint32_t* __restrict__ owner_total, const unsigned long long* __restrict__ bad, uint64_t capacity,
                                 uint32_t* __restrict__ row) {
  const uint32_t i = threadIdx.x;
  if (i < (uint32_t)kMaxRanks) row[i] = owner_total[i];
  if (i == 0) {
    row[kMaxRanks] = (uint32_t)capacity; row[kMaxRanks + 1] = (uint32_t)(capacity >> 32);
    const unsigned long long b = *bad;
    row[kMaxRanks + 2] = b > 0xffffffffull ? 0xffffffffu : (uint32_t)b; row[kMaxRanks + 3] = 0;
  }
}

// ---------------------------------------------------------------- K4: count
// hist[owner * nblocks + block] = records of this block owned by `owner`
__global__ void __launch_bounds__(kRouteThreads) route_count_kernel(const uint8_t* __restrict__ rec, uint64_t n, uint64_t n_global,
                                                                    const uint8_t* __restrict__ owner_of, uint32_t nranks,
                                                                    uint32_t* __restrict__ hist, uint32_t nblocks,
                                                                    unsigned long long* __restrict__ bad) {
  __shared__ uint32_t h[kMaxRanks];
  if (threadIdx.x < kMaxRanks) h[threadIdx.x] = 0;
  __syncthreads();
  const uint64_t base = (uint64_t)blockIdx.x * kRouteBlockRecs;
  constexpr int kIts = kRouteBlockRecs / kRouteThreads;
  // all loads of a thread's 8 records first (independent, in flight together), then the owner lookups, then the votes
  unsigned long long g[kIts];
#pragma unroll
  for (int it = 0; it < kIts; ++it) {
    const uint64_t i = base + (uint64_t)it * kRouteThreads + threadIdx.x;
    g[it] = i < n ? *reinterpret_cast<const unsigned long long*>(rec + i * 64 + 8) : ~0ull;
  }
  uint32_t o[kIts];
#pragma unroll
  for (int it = 0; it < kIts; ++it) {
    const uint64_t i = base + (uint64_t)it * kRouteThreads + threadIdx.x;
    o[it] = 0xffffffffu;
    if (i < n) { if (g[it] < n_global) o[it] = owner_of[g[it]]; else atomicAdd(bad, 1ull); }
  }
#pragma unroll
  for (int it = 0; it < kIts; ++it) {
    // one atomic per (warp, owner)
    for (uint32_t r = 0; r < nranks; ++r) {
      const uint32_t m = __ballot_sync(0xffffffffu, o[it] == r);
      if ((threadIdx.x & 31) == 0 && m) atomicAdd(&h[r], __popc(m));
    }
  }
  __syncthreads();
  if (threadIdx.x < nranks) hist[threadIdx.x * nblocks + blockIdx.x] = h[threadIdx.x];
}

// ---------------------------------------------------------------- K4: stable scatter
// dst[r] is where this rank's records for owner r start (local send region or the owner's receive buffer
// through a peer mapping); block_base[owner * nblocks + block] = exclusive scan of hist within each owner.
struct RouteDst { uint8_t* p[kMaxRanks]; };

__global__ void __launch_bounds__(kRouteThreads) route_scatter_kernel(const uint8_t* __restrict__ rec, uint64_t n, uint64_t n_global,
                                                                      const uint8_t* __restrict__ owner_of, const uint32_t* __restrict__ local_of,
                                                                      uint32_t nranks, const uint32_t* __restrict__ block_base, uint32_t nblocks,
                                                                      const uint32_t* __restrict__ owner_total_ex, RouteDst dst) {
  __shared__ uint32_t run[kMaxRanks];                       // next free slot per owner inside this block's range
  __shared__ uint32_t wcnt[kRouteThreads / 32][kMaxRanks];  // per-warp counts of the current round
  __shared__ uint32_t dpos[kRouteThreads];                  // destination record index (within the owner's region) of each record
  __shared__ uint8_t down[kRouteThreads];
  __shared__ uint32_t dloc[kRouteThreads];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x < nranks) run[threadIdx.x] = block_base[threadIdx.x * nblocks + blockIdx.x] - owner_total_ex[threadIdx.x];  // relative to the owner's region
  __syncthreads();
  const uint64_t base = (uint64_t)blockIdx.x * kRouteBlockRecs;
  for (int it = 0; it < kRouteBlockRecs / kRouteThreads; ++it) {
    const uint64_t i = base + (uint64_t)it * kRouteThreads + threadIdx.x;
    uint32_t o = 0xffffffffu, loc = 0;
    if (i < n) {
      const unsigned long long g = *reinterpret_cast<const unsigned long long*>(rec + i * 64 + 8);
      if (g < n_global) { o = owner_of[g]; loc = local_of[g]; }
    }
    // stable rank: records with the same owner in lower lanes of this warp, earlier warps, earlier rounds
    uint32_t rank_in_warp = 0;
    for (uint32_t r = 0; r < nranks; ++r) {
      const uint32_t m = __ballot_sync(0xffffffffu, o == r);
      if (o == r) rank_in_warp = __popc(m & ((1u << lane) - 1u));
      if (lane == 0) wcnt[warp][r] = __popc(m);
    }
    __syncthreads();
    uint32_t before = 0;
    if (o != 0xffffffffu) {
      for (int w = 0; w < warp; ++w) before += wcnt[w][o];
      dpos[threadIdx.x] = run[o] + before + rank_in_warp;
    }
    down[threadIdx.x] = (uint8_t)(o == 0xffffffffu ? 0xff : o);
    dloc[threadIdx.x] = loc;
    __syncthreads();
    if (threadIdx.x < nranks) {
      uint32_t tot = 0;
      for (int w = 0; w < kRouteThreads / 32; ++w) tot += wcnt[w][threadIdx.x];
      run[threadIdx.x] += tot;
    }
    // copy: 4 lanes x 16 B per record, 64 records per pass
    for (int pass = 0; pass < 4; ++pass) {
      const int rl = pass * 64 + (threadIdx.x >> 2);  // record within the round
      const int part = threadIdx.x & 3;
      const uint64_t src_i = base + (uint64_t)it * kRouteThreads + rl;
      const uint8_t ow = down[rl];
      if (src_i < n && ow != 0xff) {
        uint4 v = __ldg(reinterpret_cast<const uint4*>(rec + src_i * 64) + part);
        if (part == 0) { v.z = dloc[rl]; v.w = 0u; }  // agg field := the owner's LOCAL aggregate index
        reinterpret_cast<uint4*>(dst.p[ow] + (uint64_t)dpos[rl] * 64)[part] = v;
      }
    }
    __syncthreads();
  }
}

// after the device-wide exclusive scan of hist (row-major [owner][block], one zero row appended): row r starts at
// hist[r * nblocks]; per-owner totals are differences of consecutive row starts
__global__ void route_totals_kernel(const uint32_t* __restrict__ hist, uint32_t nblocks, uint32_t* __restrict__ owner_total,
                                    uint32_t* __restrict__ owner_total_ex) {
  const uint32_t r = threadIdx.x;
  if (r < (uint32_t)kMaxRanks) {
    const uint32_t s0 = hist[(size_t)r * nblocks], s1 = hist[(size_t)(r + 1) * nblocks];
    owner_total_ex[r] = s0;
    owner_total[r] = s1 - s0;
  }
}

inline uint32_t cdiv64(uint64_t a, uint32_t b) { return (uint32_t)((a + b - 1) / b); }

}  // namespace

// ---------------------------------------------------------------- NCCL through dlopen (no link-time dependency)
bool NcclApi::load(std::string* err) {
  if (lib) return true;
  lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!lib) lib = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  if (!lib) { *err = std::string("dlopen libnccl.so.2: ") + dlerror(); return false; }
#define SGR_SYM(field, name) *(void**)(&field) = dlsym(lib, name); if (!field) { *err = std::string("missing symbol ") + name; return false; }
  SGR_SYM(GetUniqueId, "ncclGetUniqueId") SGR_SYM(CommInitRank, "ncclCommInitRank") SGR_SYM(CommDestroy, "ncclCommDestroy")
  SGR_SYM(GroupStart, "ncclGroupStart") SGR_SYM(GroupEnd, "ncclGroupEnd") SGR_SYM(Send, "ncclSend") SGR_SYM(Recv, "ncclRecv")
  SGR_SYM(AllGather, "ncclAllGather") SGR_SYM(GetErrorString, "ncclGetErrorString")
#undef SGR_SYM
  return true;
}
NcclApi& nccl_api() { static NcclApi api; return api; }
#define g_nccl (nccl_api())

DistState* dist_create() { return new DistState(); }

void dist_destroy(DistState* d) {
  if (!d) return;
  for (void* p : d->opened) cudaIpcCloseMemHandle(p);
  if (d->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(d->comm);
  d->owner_of.release(); d->local_of.release(); d->global_of_local.release(); d->part_tmp.release(); d->flags.release();
  d->pos.release(); d->scan_tmp.release(); d->hist.release(); d->owner_total.release(); d->counts_all.release();
  d->send_buf.release(); d->recv_buf.release();
  d->route_of.release(); d->lb.release(); d->push_ctl.release(); d->gather_buf.release();
  if (d->stream2) cudaStreamDestroy(d->stream2);
  if (d->stream_hi) cudaStreamDestroy(d->stream_hi);
  if (d->h_pinned) cudaFreeHost(d->h_pinned);
  for (auto& e : d->pev) if (e) cudaEventDestroy(e);
  for (auto& e : d->ev) if (e) cudaEventDestroy(e);
  delete d;
}

int dist_unique_id(void* out128, std::string* err) {
  if (!g_nccl.load(err)) return SGR_ERR_DIST;
  ncclUniqueId id;
  ncclResult_t r = g_nccl.GetUniqueId(&id);
  if (r != ncclSuccess) { *err = std::string("ncclGetUniqueId: ") + g_nccl.GetErrorString(r); return SGR_ERR_DIST; }
  static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
  memcpy(out128, &id, 128);
  return SGR_OK;
}

int dist_init(DistState* d, int rank, int nranks, const void* unique_id, uint64_t recv_capacity_records, cudaStream_t st, std::string* err) {
  if (nranks < 1 || nranks > kMaxRanks || rank < 0 || rank >= nranks) { *err = "rank/nranks out of range"; return SGR_ERR_INVALID; }
  d->rank = rank; d->nranks = nranks; d->recv_capacity = recv_capacity_records;
  d->loopback = nranks > 1 && !unique_id;   // ranks of one process (tests): peers arrive through dist_set_peers, barriers are the caller's
  for (auto& e : d->ev) if (!e && cudaEventCreate(&e) != cudaSuccess) { *err = "cudaEventCreate"; return SGR_ERR_CUDA; }
  for (auto& e : d->pev) if (!e && cudaEventCreate(&e) != cudaSuccess) { *err = "cudaEventCreate"; return SGR_ERR_CUDA; }
  if (!d->stream2) {
    int lo = 0, hi = 0;
    cudaDeviceGetStreamPriorityRange(&lo, &hi);
    if (cudaStreamCreateWithPriority(&d->stream2, cudaStreamNonBlocking, lo) != cudaSuccess ||
        cudaStreamCreateWithPriority(&d->stream_hi, cudaStreamNonBlocking, hi) != cudaSuccess) { *err = "cudaStreamCreate"; return SGR_ERR_CUDA; }
  }
  if (nranks > 1 && !d->loopback) {
    if (!g_nccl.load(err)) return SGR_ERR_DIST;
    ncclUniqueId id; memcpy(&id, unique_id, 128);
    ncclResult_t r = g_nccl.CommInitRank(&d->comm, nranks, id, rank);
    if (r != ncclSuccess) { *err = std::string("ncclCommInitRank: ") + g_nccl.GetErrorString(r); return SGR_ERR_DIST; }
  }
  const size_t rec_bytes = (nranks > 1 || recv_capacity_records) ? recv_capacity_records * 64 : 0;
  cudaError_t ce = d->recv_buf.reserve(kRecvHeaderBytes + rec_bytes);
  if (ce != cudaSuccess) { *err = std::string("receive buffer: ") + cudaGetErrorString(ce); return SGR_ERR_OOM; }
  if ((ce = cudaMemsetAsync(d->recv_buf.p, 0, kRecvHeaderBytes, st)) != cudaSuccess || (ce = cudaStreamSynchronize(st)) != cudaSuccess) {
    *err = std::string("receive header: ") + cudaGetErrorString(ce); return SGR_ERR_CUDA;
  }
  d->peer_base[rank] = (uint8_t*)d->recv_buf.p;
  d->peer_recv[rank] = (uint8_t*)d->recv_buf.p + kRecvHeaderBytes;
  d->epoch = 0;
  return SGR_OK;
}

int dist_ipc_export(DistState* d, void* out64, std::string* err) {
  cudaIpcMemHandle_t h;
  cudaError_t ce = cudaIpcGetMemHandle(&h, d->recv_buf.p);
  if (ce != cudaSuccess) { *err = std::string("cudaIpcGetMemHandle: ") + cudaGetErrorString(ce); return SGR_ERR_CUDA; }
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "ipc handle is 64 bytes");
  memcpy(out64, &h, 64);
  return SGR_OK;
}

int dist_ipc_import(DistState* d, const void* handles, std::string* err) {
  for (int r = 0; r < d->nranks; ++r) {
    if (r == d->rank) continue;
    cudaIpcMemHandle_t h; memcpy(&h, (const uint8_t*)handles + (size_t)r * 64, 64);
    void* p = nullptr;
    cudaError_t ce = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
    if (ce != cudaSuccess) { *err = std::string("cudaIpcOpenMemHandle(rank ") + std::to_string(r) + "): " + cudaGetErrorString(ce); return SGR_ERR_DIST; }
    d->peer_base[r] = (uint8_t*)p;
    d->peer_recv[r] = (uint8_t*)p + kRecvHeaderBytes;
    d->opened.push_back(p);
  }
  d->peers_mapped = true;
  return SGR_OK;
}

bool LoopbackGroup::arrive_and_wait(int seconds) {
  std::unique_lock<std::mutex> l(mu);
  const uint64_t gen = generation;
  if (++arrived == nranks) { arrived = 0; ++generation; cv.notify_all(); return true; }
  if (cv.wait_for(l, std::chrono::seconds(seconds), [&] { return generation != gen; })) return true;
  --arrived;
  return false;
}

// the group of the loopback ranks whose rank 0 owns receive allocation `key` (one group per live job)
static std::shared_ptr<LoopbackGroup> loopback_group(const void* key, int nranks) {
  static std::mutex mu;
  static std::map<const void*, std::weak_ptr<LoopbackGroup>> groups;
  std::lock_guard<std::mutex> l(mu);
  std::shared_ptr<LoopbackGroup> g = groups[key].lock();
  if (!g || g->nranks != nranks) {
    g = std::make_shared<LoopbackGroup>();
    g->nranks = nranks;
    groups[key] = g;
  }
  return g;
}

// loopback ranks (one process, one device): the other ranks' receive allocations as plain device pointers
int dist_set_peers(DistState* d, void* const* bases, std::string* err) {
  if (!d->loopback) { *err = "sgr_dist_set_peers is for loopback ranks (sgr_dist_init without a unique id)"; return SGR_ERR_INVALID; }
  for (int r = 0; r < d->nranks; ++r) {
    if (r == d->rank) continue;
    if (!bases[r]) { *err = "null peer base"; return SGR_ERR_INVALID; }
    d->peer_base[r] = (uint8_t*)bases[r];
    d->peer_recv[r] = (uint8_t*)bases[r] + kRecvHeaderBytes;
  }
  d->group = loopback_group(d->peer_base[0], d->nranks);
  d->peers_mapped = true;
  return SGR_OK;
}
void* dist_recv_base(const DistState* d) { return d->recv_buf.p; }

int dist_set_partitions(DistState* d, const uint32_t* partition_of_agg, uint64_t n_global, cudaStream_t st, std::string* err) {
  if (n_global >= (1ull << 32)) { *err = "at most 2^32 global aggregates"; return SGR_ERR_UNSUPPORTED; }
  cudaError_t ce;
  DTRY(d->part_tmp.reserve(n_global * 4)); DTRY(d->owner_of.reserve(n_global)); DTRY(d->local_of.reserve(n_global * 4));
  DTRY(d->flags.reserve(n_global * 4)); DTRY(d->pos.reserve(n_global * 4));
  DTRY(cudaMemcpyAsync(d->part_tmp.p, partition_of_agg, n_global * 4, cudaMemcpyHostToDevice, st));
  const uint32_t nb = cdiv64(n_global, 256);
  owner_table_kernel<<<nb, 256, 0, st>>>((const uint32_t*)d->part_tmp.p, n_global, (uint32_t)d->nranks, (uint8_t*)d->owner_of.p);
  // local index = rank of the aggregate among those with the same owner (ascending global index)
  uint64_t n_local = 0;
  for (int r = 0; r < d->nranks; ++r) {
    owner_flags_kernel<<<nb, 256, 0, st>>>((const uint8_t*)d->owner_of.p, n_global, (uint32_t)r, (uint32_t*)d->flags.p);
    DTRY(exclusive_sum_u32((const uint32_t*)d->flags.p, (uint32_t*)d->pos.p, (uint32_t)n_global, d->scan_tmp, st));
    if (r == d->rank) {
      uint32_t last_pos = 0, last_flag = 0;
      if (n_global) {
        DTRY(cudaMemcpyAsync(&last_pos, (uint32_t*)d->pos.p + n_global - 1, 4, cudaMemcpyDeviceToHost, st));
        DTRY(cudaMemcpyAsync(&last_flag, (uint32_t*)d->flags.p + n_global - 1, 4, cudaMemcpyDeviceToHost, st));
        DTRY(cudaStreamSynchronize(st));
      }
      n_local = (uint64_t)last_pos + last_flag;
      DTRY(d->global_of_local.reserve((n_local + 1) * 4));
    }
    local_index_kernel<<<nb, 256, 0, st>>>((const uint8_t*)d->owner_of.p, n_global, (uint32_t)r, (const uint32_t*)d->pos.p,
                                           (uint32_t*)d->local_of.p, (uint32_t*)d->global_of_local.p, (uint32_t)d->rank);
  }
  // owner << 28 | local index in one word: one lookup per record in the push kernel (route_push.cu)
  // (the push path is taken only while n_global <= 2^28, so every local index fits its 28 bits)
  DTRY(d->route_of.reserve(n_global * 4 + 4));
  route_table_kernel<<<nb, 256, 0, st>>>((const uint8_t*)d->owner_of.p, (const uint32_t*)d->local_of.p, n_global, (uint32_t*)d->route_of.p);
  DTRY(cudaStreamSynchronize(st));
  d->n_global = n_global; d->n_local = n_local;
  return SGR_OK;
}

uint64_t dist_n_local(const DistState* d) { return d->n_local; }
uint64_t dist_n_global(const DistState* d) { return d->n_global; }
int dist_nranks(const DistState* d) { return d->nranks; }
bool dist_is_loopback(const DistState* d) { return d->loopback; }
void dist_clear_stats(DistState* d, uint64_t n_records) { d->stats = DistStats{}; d->stats.n_sent = n_records; d->stats.n_recv = n_records; }
const uint32_t* dist_global_of_local(const DistState* d) { return (const uint32_t*)d->global_of_local.p; }
const DistStats* dist_stats(const DistState* d) { return &d->stats; }
const uint8_t* dist_recv_buffer(const DistState* d) { return d->peer_recv[d->rank]; }

// Route this rank's records to their owners. On return (stream-ordered) the receive buffer holds n_recv records,
// grouped by source rank, each with its agg field rewritten to the local aggregate index.
int dist_route(DistState* d, const uint8_t* d_records, uint64_t n, bool fused, unsigned long long* d_counters, cudaStream_t st,
               uint64_t* n_recv_out, std::string* err) {
  cudaError_t ce;
  if (!d->n_global) { *err = "no partition table: call sgr_dist_set_partitions first"; return SGR_ERR_NOT_LOADED; }
  if (d->loopback) { *err = "loopback ranks have no NCCL communicator: use fused >= 2 with a sort-free program"; return SGR_ERR_UNSUPPORTED; }
  if (n >= (1ull << 32)) { *err = "at most 2^32 records per rank per exchange"; return SGR_ERR_UNSUPPORTED; }
  if (fused && d->nranks > 1 && !d->peers_mapped) { *err = "fused route needs the peers' receive buffers (sgr_dist_ipc_import)"; return SGR_ERR_NOT_LOADED; }
  const int R = d->nranks;
  const uint32_t nblocks = n ? cdiv64(n, kRouteBlockRecs) : 1;
  DTRY(d->hist.reserve((size_t)(kMaxRanks + 1) * nblocks * 4 + 64));
  DTRY(d->owner_total.reserve(2 * kMaxRanks * 4));
  uint32_t* owner_total = (uint32_t*)d->owner_total.p;
  uint32_t* owner_total_ex = owner_total + kMaxRanks;

  DTRY(cudaEventRecord(d->ev[0], st));
  DTRY(cudaMemsetAsync(d_counters, 0, 64, st));
  DTRY(cudaMemsetAsync(d->hist.p, 0, (size_t)(kMaxRanks + 1) * nblocks * 4 + 64, st));
  if (n) route_count_kernel<<<nblocks, kRouteThreads, 0, st>>>(d_records, n, d->n_global, (const uint8_t*)d->owner_of.p, (uint32_t)R,
                                                               (uint32_t*)d->hist.p, nblocks, d_counters + 4);
  DTRY(exclusive_sum_u32((const uint32_t*)d->hist.p, (uint32_t*)d->hist.p, (uint32_t)((size_t)kMaxRanks * nblocks + 1), d->scan_tmp, st));
  route_totals_kernel<<<1, 32, 0, st>>>((const uint32_t*)d->hist.p, nblocks, owner_total, owner_total_ex);
  DTRY(cudaGetLastError());
  DTRY(cudaEventRecord(d->ev[1], st));

  // ---- counts: send[r] on every rank -> nranks x nranks matrix on every rank. Each row also carries the rank's receive capacity
  //      and its count of bad records, so that EVERY rank evaluates EVERY rank's outcome and all fail (or proceed) together,
  //      before anything is written into a peer: a rank over capacity is never written past, nobody is left alone in a collective
  constexpr int kRow = kMaxRanks + 4;   // counts | capacity lo, hi | bad | pad
  DTRY(d->counts_all.reserve((size_t)(kMaxRanks + 1) * kRow * 4 + 64));
  uint32_t* d_row = (uint32_t*)d->counts_all.p;                 // my row
  uint32_t* d_all = d_row + kRow;                               // the gathered matrix
  route_row_kernel<<<1, 32, 0, st>>>(owner_total, d_counters + 4, d->recv_capacity, d_row);
  std::vector<uint32_t> send_cnt(kMaxRanks, 0);
  std::vector<uint32_t> rows((size_t)R * kRow, 0);
  if (R > 1) {
    NTRY(g_nccl.AllGather(d_row, d_all, kRow, ncclUint32, d->comm, st));
    DTRY(cudaMemcpyAsync(rows.data(), d_all, (size_t)R * kRow * 4, cudaMemcpyDeviceToHost, st));
  } else {
    DTRY(cudaMemcpyAsync(rows.data(), d_row, kRow * 4, cudaMemcpyDeviceToHost, st));
  }
  DTRY(cudaStreamSynchronize(st));
  std::vector<uint32_t> all_cnt((size_t)R * kMaxRanks, 0);
  for (int s = 0; s < R; ++s) for (int q = 0; q < kMaxRanks; ++q) all_cnt[(size_t)s * kMaxRanks + q] = rows[(size_t)s * kRow + q];
  for (int s = 0; s < R; ++s)
    if (rows[(size_t)s * kRow + kMaxRanks + 2]) {
      *err = "rank " + std::to_string(s) + ": " + std::to_string(rows[(size_t)s * kRow + kMaxRanks + 2]) + "+ records carry a global aggregate index >= n_global";
      return SGR_ERR_INVALID;
    }
  for (int r = 0; r < R; ++r) send_cnt[r] = all_cnt[(size_t)d->rank * kMaxRanks + r];
  // receive layout on rank q: blocks by source rank s, in rank order
  uint64_t n_recv = 0;
  std::vector<uint64_t> recv_off(R, 0);
  for (int s = 0; s < R; ++s) { recv_off[s] = n_recv; n_recv += all_cnt[(size_t)s * kMaxRanks + d->rank]; }
  for (int q = 0; q < R; ++q) {
    uint64_t nq = 0;
    for (int s = 0; s < R; ++s) nq += all_cnt[(size_t)s * kMaxRanks + q];
    const uint64_t capq = ((uint64_t)rows[(size_t)q * kRow + kMaxRanks + 1] << 32) | rows[(size_t)q * kRow + kMaxRanks];
    if (nq > capq) {
      *err = "receive buffer of rank " + std::to_string(q) + " too small: " + std::to_string(nq) + " > " + std::to_string(capq) + " records";
      return SGR_ERR_CAPACITY;
    }
  }
  *n_recv_out = n_recv;
  DTRY(cudaEventRecord(d->ev[2], st));

  // ---- scatter, straight to the destination
  RouteDst dst{};
  if (fused) {
    // my block inside owner q's receive buffer starts after the blocks of the ranks before me
    for (int q = 0; q < R; ++q) {
      uint64_t off = 0;
      for (int s = 0; s < d->rank; ++s) off += all_cnt[(size_t)s * kMaxRanks + q];
      dst.p[q] = d->peer_recv[q] + off * 64;
    }
  } else {
    DTRY(d->send_buf.reserve(n * 64));
    uint64_t off = 0;
    for (int q = 0; q < R; ++q) { dst.p[q] = (uint8_t*)d->send_buf.p + off * 64; off += send_cnt[q]; }
    if (R == 1) dst.p[0] = d->peer_recv[d->rank];
  }
  if (n) route_scatter_kernel<<<nblocks, kRouteThreads, 0, st>>>(d_records, n, d->n_global, (const uint8_t*)d->owner_of.p,
                                                                 (const uint32_t*)d->local_of.p, (uint32_t)R, (const uint32_t*)d->hist.p,
                                                                 nblocks, owner_total_ex, dst);
  DTRY(cudaGetLastError());
  DTRY(cudaEventRecord(d->ev[3], st));
  if (R > 1) {
    if (fused) {
      // every source has to be done before anyone folds: a 4-byte all-gather is the stream-ordered barrier
      NTRY(g_nccl.AllGather(owner_total, d->counts_all.p, 1, ncclUint32, d->comm, st));
    } else {
      NTRY(g_nccl.GroupStart());
      uint64_t off = 0;
      for (int q = 0; q < R; ++q) {
        if (send_cnt[q]) NTRY(g_nccl.Send((const uint8_t*)d->send_buf.p + off * 64, (size_t)send_cnt[q] * 64, ncclUint8, q, d->comm, st));
        off += send_cnt[q];
        const uint64_t rc = all_cnt[(size_t)q * kMaxRanks + d->rank];
        if (rc) NTRY(g_nccl.Recv(d->peer_recv[d->rank] + recv_off[q] * 64, (size_t)rc * 64, ncclUint8, q, d->comm, st));
      }
      NTRY(g_nccl.GroupEnd());
    }
  }
  DTRY(cudaEventRecord(d->ev[4], st));
  DTRY(cudaStreamSynchronize(st));
  float a = 0, b = 0, c = 0, e2 = 0;
  cudaEventElapsedTime(&a, d->ev[0], d->ev[1]); cudaEventElapsedTime(&b, d->ev[1], d->ev[2]);
  cudaEventElapsedTime(&c, d->ev[2], d->ev[3]); cudaEventElapsedTime(&e2, d->ev[3], d->ev[4]);
  d->stats.ms_count = a; d->stats.ms_counts_exchange = b; d->stats.ms_scatter = c; d->stats.ms_exchange = e2;
  d->stats.n_sent = n; d->stats.n_recv = n_recv;
  uint64_t remote = 0;
  for (int q = 0; q < R; ++q) if (q != d->rank) remote += send_cnt[q];
  d->stats.n_sent_remote = remote;
  return SGR_OK;
}

}  // namespace sgr
