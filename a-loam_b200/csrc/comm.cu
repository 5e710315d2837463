// Multi-GPU scan-to-map (SURVEY.md 8e): one process per GPU, the submap is split into spatial slabs (+ one-cell halo),
// every rank fits only the stack points whose cell it owns and the ranks meet in ONE collective per evaluation:
// all-reduce (sum) of 32 doubles = [J^T J upper 21 | J^T r 6 | cost | #edge | #plane | pad] over NVLink / NVSwitch: inside the
// solve kernel through peer memory when the ranks can map each other's, else ncclAllReduce between per-evaluation kernels.
// Every rank then takes the identical trust-region step -- no broadcast, no host round trip.  launch_lm_batch (below) issues
// every LM solve of the library, local or exchanged.
//
// NCCL is loaded with dlopen at communicator creation, so libaloam_b200.so itself has no NCCL dependency and loads on a
// CPU-only box; inside a torch process the already-loaded torch-bundled libnccl.so.2 is picked up by soname.
#include <dlfcn.h>
#include <nccl.h>
#include "ctx.h"

using namespace aloam;

namespace {
struct NcclApi {
  void* handle = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
};
NcclApi g_nccl;

bool load_nccl() {
  if (g_nccl.handle) return true;
  void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  if (!h) { fprintf(stderr, "[aloam_b200] cannot load libnccl: %s\n", dlerror()); return false; }
  g_nccl.GetUniqueId = (decltype(g_nccl.GetUniqueId))dlsym(h, "ncclGetUniqueId");
  g_nccl.CommInitRank = (decltype(g_nccl.CommInitRank))dlsym(h, "ncclCommInitRank");
  g_nccl.AllReduce = (decltype(g_nccl.AllReduce))dlsym(h, "ncclAllReduce");
  g_nccl.AllGather = (decltype(g_nccl.AllGather))dlsym(h, "ncclAllGather");
  g_nccl.CommDestroy = (decltype(g_nccl.CommDestroy))dlsym(h, "ncclCommDestroy");
  g_nccl.GetErrorString = (decltype(g_nccl.GetErrorString))dlsym(h, "ncclGetErrorString");
  if (!g_nccl.GetUniqueId || !g_nccl.CommInitRank || !g_nccl.AllReduce || !g_nccl.CommDestroy) return false;
  g_nccl.handle = h;
  return true;
}
}  // namespace

// peer-memory exchange state of a context (see PeerX, kernels.h)
struct PeerState {
  PeerX px = {};
  void* own = nullptr;                 // this rank's mailbox allocation (boxes, counter, totals, error word)
  void* opened[ALOAM_MAX_RANKS] = {};  // peers' mailboxes mapped into this process (cudaIpcOpenMemHandle)
  int poison = 0;                      // test hook: the next peer_err_reset writes 1 instead of 0
};

// a rank's mailbox allocation in a world of `world` ranks: boxes [2 parities][world][32][2] words, the evaluation counter (64 B),
// the totals [2][32] and the error word (64 B)
static size_t mailbox_box_bytes(int world) { return (size_t)2 * world * 32 * 2 * sizeof(unsigned long long); }
static size_t mailbox_bytes(int world) { return mailbox_box_bytes(world) + 64 + 2 * 32 * sizeof(double) + 64; }
// points the counter, totals and error word of ps->px into this rank's own (zeroed) mailbox
static void mailbox_locals(PeerState* ps, int rank, int world) {
  char* mbox = static_cast<char*>(ps->own) + mailbox_box_bytes(world);
  ps->px.seq = reinterpret_cast<unsigned long long*>(mbox);
  ps->px.gtot = reinterpret_cast<double*>(mbox + 64);
  ps->px.err = reinterpret_cast<int*>(mbox + 64 + 2 * 32 * sizeof(double));
  ps->px.rank = rank; ps->px.world = world;
}

// unmaps the peers' mailboxes, frees this rank's and forgets the peer state (back to the NCCL path)
static void peer_drop(aloam_ctx* c) {
  PeerState* ps = static_cast<PeerState*>(c->peer);
  if (!ps) return;
  for (void* p : ps->opened) if (p) cudaIpcCloseMemHandle(p);
  if (ps->own) cudaFree(ps->own);
  delete ps;
  c->peer = nullptr;
}

// a device buffer that lives for one call
template <typename T> struct DeviceTemp {
  T* p = nullptr;
  ~DeviceTemp() { if (p) cudaFree(p); }
};

// Sum of `count` elements of `type` (ncclDouble or ncclInt32) over the ranks, src -> dst on c->stream (in place when they are
// equal): ncclAllReduce on a communicator; on a context that emulates a rank the sum over its one rank, a device copy.
int comm_allreduce(aloam_ctx* c, const void* src, void* dst, size_t count, ncclDataType_t type) {
  if (!c->comm) {
    if (src != dst) CUDA_CHECK_RET(cudaMemcpyAsync(dst, src, count * (type == ncclDouble ? sizeof(double) : sizeof(int)), cudaMemcpyDeviceToDevice, c->stream));
    return ALOAM_OK;
  }
  const ncclResult_t r = g_nccl.AllReduce(src, dst, count, type, ncclSum, (ncclComm_t)c->comm, c->stream);
  if (r != ncclSuccess) { fprintf(stderr, "[aloam_b200] ncclAllReduce failed: %s\n", g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "?"); return ALOAM_ERR_COMM; }
  return ALOAM_OK;
}

int launch_lm_batch(aloam_ctx* c, bool pdl, const Batch<LmArgs>& args, int lanes, const LmParams& lp, int mode, int integrate, bool general,
                    bool exchange) {
  const dim3 grid(kLmCluster, lanes), block(ALOAM_LM_THREADS);
  const size_t smem = lm_dynamic_smem_bytes();
  if (!exchange) {
    if (general) launch_ex(c, KID_LM_SOLVE, k_lm_solve_x, grid, block, smem, kLmCluster, pdl, args, lp, mode, integrate, PeerX{});
    else launch_ex(c, KID_LM_SOLVE, k_lm_solve, grid, block, smem, kLmCluster, pdl, args, lp, mode, integrate);
    return ALOAM_OK;
  }
  if (lanes != 1) return ALOAM_ERR_STATE;   // the ranks solve one trajectory together
  if (const PeerState* ps = static_cast<const PeerState*>(c->peer)) {
    // ONE launch per solve: the cluster kernel of the single-GPU path with the all-reduce of every evaluation done inside it
    // over NVLink peer memory; early termination ends the solve on every rank at the same evaluation
    launch_ex(c, KID_LM_SOLVE, k_lm_solve_x, grid, block, smem, kLmCluster, pdl, args, lp, mode, integrate, ps->px);
    return ALOAM_OK;
  }
  // per evaluation: this rank's blocks, the all-reduce, the step (lm.cu, "Sharded solve")
  const LmArgs& a = args.a[0];
  double* local = c->d_lm_tot + 32;
  for (int e = 0; e <= lp.max_iters; ++e) {
    const int first = e == 0;
    launch_ex(c, KID_LM_SHARD, k_lm_eval_shard, dim3(kLmCluster), block, smem, kLmCluster, false, a.blocks, a.n_blocks_ptr, a.n_blocks_host,
              a.x7, c->d_lm_state, first, lp.huber_a, local);
    const int rc = comm_allreduce(c, local, c->d_lm_tot, 32, ncclDouble);
    if (rc) return rc;
    LAUNCH(c, KID_LM_SHARD, k_lm_tr_shard, 1, 32, 0, c->d_lm_state, (const double*)c->d_lm_tot, a.x7, first, lp, a.summary);
  }
  return ALOAM_OK;
}

// Maps every rank's mailbox into every other rank (CUDA IPC handles exchanged with one ncclAllGather).  Returns false (and leaves
// the NCCL path in place) when peer access is not available or ALOAM_NO_PEER is set.
static bool peer_setup(aloam_ctx* c, int rank, int world) {
  if (getenv("ALOAM_NO_PEER") || world > ALOAM_MAX_RANKS || !g_nccl.AllGather) return false;
  PeerState* ps = new (std::nothrow) PeerState();
  if (!ps) return false;
  c->peer = ps;
  const size_t total = mailbox_bytes(world);
  bool ok = cudaMalloc(&ps->own, total) == cudaSuccess && cudaMemset(ps->own, 0, total) == cudaSuccess;
  cudaIpcMemHandle_t mine;
  ok = ok && cudaIpcGetMemHandle(&mine, ps->own) == cudaSuccess;
  DeviceTemp<cudaIpcMemHandle_t> d_all;
  std::vector<cudaIpcMemHandle_t> all(world);
  ok = ok && cudaMalloc((void**)&d_all.p, sizeof(mine) * (world + 1)) == cudaSuccess;
  // every rank must take part in the gather even if its own setup failed: a zeroed handle marks the failure
  if (!ok) std::memset(&mine, 0, sizeof(mine));
  bool gathered = false;
  if (d_all.p) {
    cudaMemcpyAsync(d_all.p + world, &mine, sizeof(mine), cudaMemcpyHostToDevice, c->stream);
    if (g_nccl.AllGather(d_all.p + world, d_all.p, sizeof(mine), ncclChar, (ncclComm_t)c->comm, c->stream) == ncclSuccess &&
        cudaMemcpyAsync(all.data(), d_all.p, sizeof(mine) * world, cudaMemcpyDeviceToHost, c->stream) == cudaSuccess &&
        cudaStreamSynchronize(c->stream) == cudaSuccess)
      gathered = true;
  }
  ok = ok && gathered;
  const cudaIpcMemHandle_t zero = {};
  for (int r = 0; r < world && ok; ++r) {
    void* base = ps->own;
    if (r != rank) {
      if (!std::memcmp(&all[r], &zero, sizeof(zero)) || cudaIpcOpenMemHandle(&ps->opened[r], all[r], cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { ok = false; break; }
      base = ps->opened[r];
    }
    ps->px.box[r] = reinterpret_cast<double*>(base);
  }
  if (!ok) {
    cudaGetLastError();
    peer_drop(c);
    fprintf(stderr, "[aloam_b200] peer-memory exchange unavailable on rank %d: the sharded LM uses ncclAllReduce\n", rank);
    return false;
  }
  mailbox_locals(ps, rank, world);
  own(c, [c] { peer_drop(c); });
  return true;
}

// what the per-evaluation solve needs beside the mailbox, created on first use: the all-reduced totals and the trust-region state
static int lm_exchange_alloc(aloam_ctx* c) {
  if (!c->d_lm_tot) CUDA_CHECK_RET(dalloc(c, &c->d_lm_tot, 64));
  if (!c->d_lm_state) CUDA_CHECK_RET(dalloc(c, reinterpret_cast<char**>(&c->d_lm_state), lm_state_bytes()));
  return ALOAM_OK;
}

int peer_err_reset(aloam_ctx* c) {
  PeerState* ps = static_cast<PeerState*>(c->peer);
  if (!ps) return ALOAM_OK;
  static const int kOne = 1;
  if (ps->poison) CUDA_CHECK_RET(cudaMemcpyAsync(ps->px.err, &kOne, sizeof(int), cudaMemcpyHostToDevice, c->stream));
  else CUDA_CHECK_RET(cudaMemsetAsync(ps->px.err, 0, sizeof(int), c->stream));
  ps->poison = 0;
  return ALOAM_OK;
}

int peer_err_fetch(aloam_ctx* c, int* dst) {
  *dst = 0;
  const PeerState* ps = static_cast<const PeerState*>(c->peer);
  if (ps) CUDA_CHECK_RET(cudaMemcpyAsync(dst, ps->px.err, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  return ALOAM_OK;
}

extern "C" {

int aloam_debug_shard_emulate(aloam_ctx* c, int rank, int world, int exchange, int poison_peer_err) {
  if (!c) return ALOAM_ERR_INVALID_ARG;
  if (c->comm) return ALOAM_ERR_STATE;
  if (world < 0 || (world > 0 && (rank < 0 || rank >= world || exchange < 0 || exchange > 2)) || (poison_peer_err && (world == 0 || exchange != 2)))
    return ALOAM_ERR_INVALID_ARG;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  if (world > 0) { const int rc = lm_exchange_alloc(c); if (rc) return rc; }   // a failure changes no setting
  if (world == 0 || exchange != 2) {
    peer_drop(c);
  } else if (!c->peer) {   // a one-rank mailbox laid out as peer_setup's, without the IPC handles and their gather
    PeerState* ps = new (std::nothrow) PeerState();
    if (!ps) return ALOAM_ERR_CUDA;
    c->peer = ps;
    own(c, [c] { peer_drop(c); });
    if (cudaMalloc(&ps->own, mailbox_bytes(1)) != cudaSuccess || cudaMemsetAsync(ps->own, 0, mailbox_bytes(1), c->stream) != cudaSuccess) {
      cudaGetLastError();
      peer_drop(c);
      return ALOAM_ERR_CUDA;
    }
    ps->px.box[0] = static_cast<double*>(ps->own);
    mailbox_locals(ps, 0, 1);
  }
  if (poison_peer_err) static_cast<PeerState*>(c->peer)->poison = 1;
  const int new_rank = world ? rank : 0, new_count = world ? world : 1;
  if (new_rank != c->shard_rank || new_count != c->shard_count) c->have_map = false;   // the map was cut for another rank
  c->shard_rank = new_rank; c->shard_count = new_count; c->shard_exchange = world ? exchange : -1;
  return ALOAM_OK;
}

// rank 0 creates the 128-byte NCCL id; the caller ships it to the other ranks (e.g. torch.distributed.broadcast)
int aloam_comm_unique_id(char out128[128]) {
  if (!out128) return ALOAM_ERR_INVALID_ARG;
  if (!load_nccl()) return ALOAM_ERR_COMM;
  ncclUniqueId id;
  if (g_nccl.GetUniqueId(&id) != ncclSuccess) return ALOAM_ERR_COMM;
  static_assert(sizeof(id) == 128, "ncclUniqueId is 128 bytes");
  std::memcpy(out128, &id, 128);
  return ALOAM_OK;
}

// joins this context to a world of `world` ranks: from now on aloam_mapping_register fits only the stack points whose
// map cell this rank owns and all-reduces the normal equations.  The uploaded map must be this rank's shard
// (owned slabs + one-cell halo; see a-loam_b200/shard.py for the host-side split).
int aloam_comm_init(aloam_ctx* c, int rank, int world, const char id128[128]) {
  if (!c || !id128 || world < 1 || rank < 0 || rank >= world) return ALOAM_ERR_INVALID_ARG;
  if (c->shard_exchange >= 0) return ALOAM_ERR_STATE;   // emulating a rank (aloam_debug_shard_emulate)
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  if (world == 1) { c->shard_rank = 0; c->shard_count = 1; return ALOAM_OK; }
  if (!load_nccl()) return ALOAM_ERR_COMM;
  ncclUniqueId id;
  std::memcpy(&id, id128, 128);
  ncclComm_t comm = nullptr;
  ncclResult_t r = g_nccl.CommInitRank(&comm, world, id, rank);
  if (r != ncclSuccess) { fprintf(stderr, "[aloam_b200] ncclCommInitRank failed: %s\n", g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "?"); return ALOAM_ERR_COMM; }
  c->comm = comm;
  own(c, [comm] { g_nccl.CommDestroy(comm); });   // an earlier communicator of this context lives on until aloam_destroy
  const int rc = lm_exchange_alloc(c); if (rc) return rc;
  c->shard_rank = rank; c->shard_count = world;
  // the 256-byte exchange of every LM evaluation goes through NVLink peer memory inside the solve kernel when the ranks can map
  // each other's memory (all ranks decide alike: the outcome of the handle exchange is the same everywhere ... see below)
  peer_drop(c);   // the peer path of an earlier communicator
  const bool mine_ok = peer_setup(c, rank, world);
  // agree on the path: one rank without peer access forces everybody onto NCCL
  DeviceTemp<int> d_flag;
  CUDA_CHECK_RET(cudaMalloc((void**)&d_flag.p, 2 * sizeof(int)));
  int h[2] = {mine_ok ? 0 : 1, 0};
  CUDA_CHECK_RET(cudaMemcpyAsync(d_flag.p, h, 8, cudaMemcpyHostToDevice, c->stream));
  if (g_nccl.AllReduce(d_flag.p, d_flag.p, 2, ncclInt32, ncclSum, (ncclComm_t)c->comm, c->stream) != ncclSuccess) return ALOAM_ERR_COMM;
  CUDA_CHECK_RET(cudaMemcpyAsync(h, d_flag.p, 8, cudaMemcpyDeviceToHost, c->stream));
  CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  if (h[0] != 0) peer_drop(c);   // somebody failed: drop the peer path here too
  return ALOAM_OK;
}

int aloam_comm_uses_peer_memory(aloam_ctx* c) { return c && c->peer ? 1 : 0; }

int aloam_shard_slab_cells(void) { return 8; }   // ownership: slab = floor((cell_x + 2^20) / 8), owner = slab mod world

}  // extern "C"
