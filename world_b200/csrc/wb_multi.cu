// wb_multi.cu -- the one exchange step of the multi-GPU path (SURVEY.md 8e): utterances are sharded over ranks
// with no data-path collective; the output arrays are reassembled on every rank by NCCL.  One process (or thread)
// per GPU; the caller moves the 128-byte NCCL id from rank 0 to the other ranks by whatever means it has (MPI,
// torch.distributed, a socket, a file) -- that is plumbing, the data path is here.
//
// NCCL is bound at RUN time (dlopen "libnccl.so.2"): the library keeps linking against cudart only, a process that
// already carries an NCCL (PyTorch's) shares it, and single-GPU users never load it.
#include "wb_internal.h"
#include <string>
#include <vector>
#include <stdint.h>

#ifndef WB_EMU
#include <dlfcn.h>
#include <nccl.h>

namespace wb {

namespace {
struct NcclApi {
  void *lib = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*Broadcast)(const void *, void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllGather)(const void *, void *, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllReduce)(const void *, void *, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  const char *(*GetErrorString)(ncclResult_t) = nullptr;
};
NcclApi g_nccl;

bool nccl_load(std::string *err) {
  if (g_nccl.lib) return true;
  const char *names[] = {"libnccl.so.2", "libnccl.so"};
  void *lib = nullptr;
  for (const char *n : names) {
    lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
    if (lib) break;
  }
  if (!lib) { *err = std::string("NCCL not found (dlopen libnccl.so.2): ") + dlerror(); return false; }
#define WB_SYM(field, name)                                                        \
  g_nccl.field = reinterpret_cast<decltype(g_nccl.field)>(dlsym(lib, name));       \
  if (!g_nccl.field) { *err = std::string("NCCL symbol missing: ") + name; return false; }
  WB_SYM(GetUniqueId, "ncclGetUniqueId")
  WB_SYM(CommInitRank, "ncclCommInitRank")
  WB_SYM(CommDestroy, "ncclCommDestroy")
  WB_SYM(Broadcast, "ncclBroadcast")
  WB_SYM(AllGather, "ncclAllGather")
  WB_SYM(AllReduce, "ncclAllReduce")
  WB_SYM(GroupStart, "ncclGroupStart")
  WB_SYM(GroupEnd, "ncclGroupEnd")
  WB_SYM(GetErrorString, "ncclGetErrorString")
#undef WB_SYM
  g_nccl.lib = lib;
  return true;
}
}  // namespace

#define WB_P2P_ARRAYS 4
struct PeerBase { unsigned char handle[64]; void *mapped; };   // one opened allocation of one peer
struct Comm {
  ncclComm_t comm = nullptr;
  int n_ranks = 1, rank = 0;
  cudaStream_t stream = nullptr;      // all collectives run here, ordered against the compute streams by events
  cudaEvent_t done = nullptr;
  // ---- peer-to-peer push path (comm_p2p_*): the other ranks' output arrays mapped through CUDA IPC
  cudaStream_t copy_stream = nullptr; // peer copies (copy engines: no SM is taken from the compute kernels)
  cudaEvent_t copy_done = nullptr;
  int *flag_dev = nullptr;            // [8] device ints for the small agreements / the closing barrier
  unsigned char *xchg_dev = nullptr;  // handle exchange buffer: [n_ranks + 1] records
  int p2p_state = 0;                  // 0 unknown, 1 usable, -1 not usable on this system (NCCL broadcasts instead)
  const void *cur_local[WB_P2P_ARRAYS] = {nullptr, nullptr, nullptr, nullptr};
  std::vector<char *> cur_peer;       // [n_ranks][WB_P2P_ARRAYS] peer addresses of the current arrays
  std::vector<std::vector<PeerBase>> opened;   // per rank: allocations opened so far
};
struct P2pRecord {                    // what a rank tells the others about its four arrays
  unsigned char handle[WB_P2P_ARRAYS][64];
  unsigned long long offset[WB_P2P_ARRAYS];
  int valid[WB_P2P_ARRAYS];
  int ok;
};

#define WB_NCCL(call, err)                                                                         \
  do {                                                                                             \
    ncclResult_t r_ = (call);                                                                      \
    if (r_ != ncclSuccess) { *(err) = std::string("NCCL: ") + g_nccl.GetErrorString(r_); return 1; } \
  } while (0)

int comm_unique_id(unsigned char *id128, std::string *err) {
  if (!nccl_load(err)) return 1;
  ncclUniqueId id;
  WB_NCCL(g_nccl.GetUniqueId(&id), err);
  static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes in every NCCL 2.x");
  memcpy(id128, &id, 128);
  return 0;
}

int comm_create(int n_ranks, int rank, const unsigned char *id128, Comm **out, std::string *err) {
  if (!nccl_load(err)) return 1;
  Comm *c = new Comm;
  c->n_ranks = n_ranks; c->rank = rank;
  ncclUniqueId id;
  memcpy(&id, id128, 128);
  ncclResult_t r = g_nccl.CommInitRank(&c->comm, n_ranks, id, rank);
  if (r != ncclSuccess) { *err = std::string("ncclCommInitRank: ") + g_nccl.GetErrorString(r); delete c; return 1; }
  // highest stream priority: when a compute kernel's CTA retires, the waiting blocks of the collective are placed
  // first -- at equal priority the blocks of the (earlier launched, 10^5-block) compute kernels keep filling the SMs
  // and the transfer only runs in their tails
  int prio_least = 0, prio_greatest = 0;
  cudaDeviceGetStreamPriorityRange(&prio_least, &prio_greatest);
  if (cudaStreamCreateWithPriority(&c->stream, cudaStreamNonBlocking, prio_greatest) != cudaSuccess ||
      cudaEventCreateWithFlags(&c->done, cudaEventDisableTiming) != cudaSuccess) {
    *err = "cannot create the communication stream";
    g_nccl.CommDestroy(c->comm);
    delete c;
    return 1;
  }
  if (cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking) != cudaSuccess ||
      cudaEventCreateWithFlags(&c->copy_done, cudaEventDisableTiming) != cudaSuccess ||
      cudaMalloc((void **)&c->flag_dev, 8 * sizeof(int)) != cudaSuccess ||
      cudaMalloc((void **)&c->xchg_dev, (size_t)(n_ranks + 1) * sizeof(P2pRecord)) != cudaSuccess) {
    cudaGetLastError();
    c->p2p_state = -1;   // the NCCL path still works
  }
  c->opened.resize(n_ranks);
  c->cur_peer.assign((size_t)n_ranks * WB_P2P_ARRAYS, nullptr);
  *out = c;
  return 0;
}

void comm_destroy(Comm *c) {
  if (!c) return;
  cudaStreamSynchronize(c->stream);
  if (c->copy_stream) cudaStreamSynchronize(c->copy_stream);
  for (auto &per_rank : c->opened)
    for (auto &pb : per_rank)
      if (pb.mapped) cudaIpcCloseMemHandle(pb.mapped);
  if (c->copy_stream) cudaStreamDestroy(c->copy_stream);
  if (c->copy_done) cudaEventDestroy(c->copy_done);
  if (c->flag_dev) cudaFree(c->flag_dev);
  if (c->xchg_dev) cudaFree(c->xchg_dev);
  if (c->comm) g_nccl.CommDestroy(c->comm);
  cudaEventDestroy(c->done);
  cudaStreamDestroy(c->stream);
  delete c;
}

int comm_ranks(const Comm *c) { return c->n_ranks; }
int comm_rank(const Comm *c) { return c->rank; }

// Rows [row0, row0 + rows) of every rank's shard: `full` is [n_ranks][rows_per_rank][row_elems]; rank r owns block r
// and its rows are already in place.  One grouped set of broadcasts (root r sends its rows, everybody else receives
// them where they belong), enqueued on the communication stream after `after` (an event on a compute stream).
int comm_gather_rows(Comm *c, double *full, size_t row_elems, size_t rows_per_rank, size_t row0, size_t rows,
                     cudaEvent_t after, std::string *err) {
  if (rows == 0 || row_elems == 0) return 0;
  if (after && cudaStreamWaitEvent(c->stream, after, 0) != cudaSuccess) { *err = "cudaStreamWaitEvent failed"; return 1; }
  if (row0 == 0 && rows == rows_per_rank) {   // whole shards: the plain in-place all-gather
    WB_NCCL(g_nccl.AllGather(full + (size_t)c->rank * rows_per_rank * row_elems, full, rows_per_rank * row_elems, ncclDouble,
                             c->comm, c->stream), err);
    return 0;
  }
  WB_NCCL(g_nccl.GroupStart(), err);
  for (int r = 0; r < c->n_ranks; ++r) {
    double *at = full + ((size_t)r * rows_per_rank + row0) * row_elems;
    ncclResult_t res = g_nccl.Broadcast(at, at, rows * row_elems, ncclDouble, r, c->comm, c->stream);
    if (res != ncclSuccess) { g_nccl.GroupEnd(); *err = std::string("ncclBroadcast: ") + g_nccl.GetErrorString(res); return 1; }
  }
  WB_NCCL(g_nccl.GroupEnd(), err);
  return 0;
}

// The same for several arrays of one utterance slice in ONE NCCL group (one fused launch instead of one per array).
int comm_gather_rows_multi(Comm *c, int n_arrays, double *const *full, const size_t *row_elems, size_t rows_per_rank,
                           size_t row0, size_t rows, cudaEvent_t after, std::string *err) {
  if (rows == 0) return 0;
  if (after && cudaStreamWaitEvent(c->stream, after, 0) != cudaSuccess) { *err = "cudaStreamWaitEvent failed"; return 1; }
  WB_NCCL(g_nccl.GroupStart(), err);
  for (int a = 0; a < n_arrays; ++a) {
    if (!full[a] || row_elems[a] == 0) continue;
    for (int r = 0; r < c->n_ranks; ++r) {
      double *at = full[a] + ((size_t)r * rows_per_rank + row0) * row_elems[a];
      ncclResult_t res = g_nccl.Broadcast(at, at, rows * row_elems[a], ncclDouble, r, c->comm, c->stream);
      if (res != ncclSuccess) { g_nccl.GroupEnd(); *err = std::string("ncclBroadcast: ") + g_nccl.GetErrorString(res); return 1; }
    }
  }
  WB_NCCL(g_nccl.GroupEnd(), err);
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// Peer-to-peer push (one process per GPU, all on one NVLink / NVSwitch node).  With NCCL the transfer of an output
// slice is a kernel on every rank: 16-32 CTAs that occupy SMs for as long as the bytes flow, taken from the compute
// (fewer channels only make the transfer the bottleneck).  Here every rank maps the other ranks' output arrays (CUDA IPC handles, exchanged
// ONCE per set of arrays through the communicator itself) and, as soon as a slice of its own rows is final, copies
// them into every peer's array with cudaMemcpyAsync on a copy stream: the copy engines move the bytes over NVLink,
// no SM is involved.  A rank only ever writes rows of its own block, so pushes never collide; one 4-byte all-reduce
// after a rank's last push closes the call (when it completes, every rank's pushes have).
// Falls back to the broadcasts when the arrays cannot be exported (memory not from cudaMalloc, no peer access).
typedef int (*wb_cuMemGetAddressRange_t)(unsigned long long *, size_t *, unsigned long long);
int comm_join(Comm *c, cudaStream_t s, std::string *err);

static bool p2p_agree(Comm *c, int local_value, int *min_out, int *max_out, std::string *err) {
  int v[2] = {local_value, -local_value};
  if (cudaMemcpyAsync(c->flag_dev, v, sizeof v, cudaMemcpyHostToDevice, c->stream) != cudaSuccess) { *err = "p2p agree: copy"; return false; }
  if (g_nccl.AllReduce(c->flag_dev, c->flag_dev + 2, 2, ncclInt, ncclMax, c->comm, c->stream) != ncclSuccess) { *err = "p2p agree: all-reduce"; return false; }
  int r[2];
  if (cudaMemcpyAsync(r, c->flag_dev + 2, sizeof r, cudaMemcpyDeviceToHost, c->stream) != cudaSuccess ||
      cudaStreamSynchronize(c->stream) != cudaSuccess) { *err = "p2p agree: sync"; return false; }
  *max_out = r[0]; *min_out = -r[1];
  return true;
}

// Makes `full[0..n_arrays)` the current arrays of the push path.  Returns 0 = usable, 1 = not usable (the caller uses
// the NCCL broadcasts), 2 = error.  Collective: every rank must call it with its own arrays at the same point.
int comm_p2p_prepare(Comm *c, int n_arrays, double *const *full, std::string *err) {
  if (c->p2p_state < 0 || n_arrays > WB_P2P_ARRAYS) return 1;
  bool same = c->p2p_state == 1;
  for (int a = 0; a < WB_P2P_ARRAYS; ++a) same = same && c->cur_local[a] == (a < n_arrays ? (const void *)full[a] : nullptr);
  int mn = 0, mx = 0;
  if (!p2p_agree(c, same ? 0 : 1, &mn, &mx, err)) return 2;
  if (mx == 0) return 0;                       // nobody's arrays changed: the mappings stand
  // ---- export this rank's arrays
  P2pRecord rec;
  memset(&rec, 0, sizeof rec);
  rec.ok = 1;
  static wb_cuMemGetAddressRange_t get_range = nullptr;
  if (!get_range) {
    void *fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuMemGetAddressRange", &fn, cudaEnableDefault, &q) == cudaSuccess && fn)
      get_range = (wb_cuMemGetAddressRange_t)fn;
  }
  for (int a = 0; a < n_arrays && rec.ok; ++a) {
    if (!full[a]) continue;
    unsigned long long base = 0; size_t size = 0;
    if (!get_range || get_range(&base, &size, (unsigned long long)(uintptr_t)full[a]) != 0) { rec.ok = 0; break; }
    cudaIpcMemHandle_t hnd;
    if (cudaIpcGetMemHandle(&hnd, (void *)(uintptr_t)base) != cudaSuccess) { cudaGetLastError(); rec.ok = 0; break; }
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
    memcpy(rec.handle[a], &hnd, 64);
    rec.offset[a] = (unsigned long long)(uintptr_t)full[a] - base;
    rec.valid[a] = 1;
  }
  // ---- everybody's records
  std::vector<P2pRecord> all((size_t)c->n_ranks);
  unsigned char *mine = c->xchg_dev + (size_t)c->n_ranks * sizeof(P2pRecord);
  if (cudaMemcpyAsync(mine, &rec, sizeof rec, cudaMemcpyHostToDevice, c->stream) != cudaSuccess ||
      g_nccl.AllGather(mine, c->xchg_dev, sizeof(P2pRecord), ncclChar, c->comm, c->stream) != ncclSuccess ||
      cudaMemcpyAsync(all.data(), c->xchg_dev, all.size() * sizeof(P2pRecord), cudaMemcpyDeviceToHost, c->stream) != cudaSuccess ||
      cudaStreamSynchronize(c->stream) != cudaSuccess) {
    *err = "p2p: handle exchange failed";
    return 2;
  }
  int ok = 1;
  for (auto &r : all) ok = ok && r.ok;
  // ---- map the peers' arrays (an allocation is opened once per peer and kept)
  std::vector<char *> peer((size_t)c->n_ranks * WB_P2P_ARRAYS, nullptr);
  for (int r = 0; r < c->n_ranks && ok; ++r) {
    if (r == c->rank) continue;
    for (int a = 0; a < n_arrays && ok; ++a) {
      if (!all[r].valid[a]) continue;
      void *mapped = nullptr;
      for (auto &pb : c->opened[r])
        if (memcmp(pb.handle, all[r].handle[a], 64) == 0) { mapped = pb.mapped; break; }
      if (!mapped) {
        cudaIpcMemHandle_t hnd;
        memcpy(&hnd, all[r].handle[a], 64);
        if (cudaIpcOpenMemHandle(&mapped, hnd, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { cudaGetLastError(); ok = 0; break; }
        PeerBase pb;
        memcpy(pb.handle, all[r].handle[a], 64);
        pb.mapped = mapped;
        c->opened[r].push_back(pb);
      }
      peer[(size_t)r * WB_P2P_ARRAYS + a] = (char *)mapped + all[r].offset[a];
    }
  }
  if (!p2p_agree(c, ok, &mn, &mx, err)) return 2;
  if (mn == 0) { c->p2p_state = -1; return 1; }   // somebody could not export or map: nobody pushes
  c->cur_peer = peer;
  for (int a = 0; a < WB_P2P_ARRAYS; ++a) c->cur_local[a] = a < n_arrays ? (const void *)full[a] : nullptr;
  c->p2p_state = 1;
  return 0;
}

// Rows [row0, row0 + rows) of this rank's block of the current arrays -> every peer, on the copy stream after `after`.
int comm_p2p_push(Comm *c, int n_arrays, const size_t *row_elems, size_t rows_per_rank, size_t row0, size_t rows,
                  cudaEvent_t after, std::string *err) {
  if (rows == 0) return 0;
  if (after && cudaStreamWaitEvent(c->copy_stream, after, 0) != cudaSuccess) { *err = "p2p: cudaStreamWaitEvent failed"; return 1; }
  for (int a = 0; a < n_arrays; ++a) {
    if (!c->cur_local[a] || row_elems[a] == 0) continue;
    const size_t off = ((size_t)c->rank * rows_per_rank + row0) * row_elems[a] * sizeof(double);
    const size_t bytes = rows * row_elems[a] * sizeof(double);
    for (int k = 1; k < c->n_ranks; ++k) {             // start with the next rank: the peers are hit evenly
      const int r = (c->rank + k) % c->n_ranks;
      char *dst = c->cur_peer[(size_t)r * WB_P2P_ARRAYS + a];
      if (!dst) continue;
      if (cudaMemcpyAsync(dst + off, (const char *)c->cur_local[a] + off, bytes, cudaMemcpyDeviceToDevice, c->copy_stream) != cudaSuccess) {
        *err = std::string("p2p: peer copy failed: ") + cudaGetErrorString(cudaGetLastError());
        return 1;
      }
    }
  }
  return 0;
}

// After the last push of a call: `s` waits until EVERY rank's pushes have landed (4-byte all-reduce behind the copies).
int comm_p2p_finish(Comm *c, cudaStream_t s, std::string *err) {
  if (cudaEventRecord(c->copy_done, c->copy_stream) != cudaSuccess ||
      cudaStreamWaitEvent(c->stream, c->copy_done, 0) != cudaSuccess) { *err = "p2p: joining the copy stream failed"; return 1; }
  WB_NCCL(g_nccl.AllReduce(c->flag_dev + 4, c->flag_dev + 5, 1, ncclInt, ncclSum, c->comm, c->stream), err);
  return comm_join(c, s, err);
}

// `s` waits for everything enqueued on the communication stream so far
int comm_join(Comm *c, cudaStream_t s, std::string *err) {
  if (cudaEventRecord(c->done, c->stream) != cudaSuccess || cudaStreamWaitEvent(s, c->done, 0) != cudaSuccess) {
    *err = "joining the communication stream failed";
    return 1;
  }
  return 0;
}

}  // namespace wb

#else   // host emulation: no devices, no NCCL -- a communicator of one rank, every call a no-op
namespace wb {
struct Comm { int n_ranks = 1, rank = 0; };
int comm_unique_id(unsigned char *id128, std::string *) { memset(id128, 0, 128); return 0; }
int comm_create(int n_ranks, int rank, const unsigned char *, Comm **out, std::string *err) {
  if (n_ranks != 1 || rank != 0) { *err = "the host emulation has no multi-GPU path"; return 1; }
  *out = new Comm;
  return 0;
}
void comm_destroy(Comm *c) { delete c; }
int comm_ranks(const Comm *c) { return c->n_ranks; }
int comm_rank(const Comm *c) { return c->rank; }
}  // namespace wb
#endif
