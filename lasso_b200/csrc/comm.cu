// lasso_b200 — multi-GPU plumbing for ONE proof sharded over G GPUs of one node (SURVEY.md §8e): one process per
// GPU.  Every polynomial of global length n >= G is partitioned by the LOW log2(G) index bits: rank g holds
// X[i*G + g].  bound_poly_var_top pairs (i, i + n/2) and both have the same low bits, so every bind and every
// round evaluation is local (src/poly/dense_mlpoly.rs:209-216, src/subprotocols/sumcheck.rs:179-237).  What is
// exchanged, and how:
//   * per sumcheck round: the (deg+1) or 3 partial sums of every rank.  NO collective and no extra launch: the
//     last CTA of the round kernel stores its tagged residues (common.cuh PubDst) straight into the receive
//     buffer of EVERY process — shared pinned host segments (POSIX shm, cudaHostRegister'ed by every process) —
//     and each of the G replicated host transcripts adds the G residues (prover.cu Ctx::fin_wait).  The round
//     trip is the single-GPU one; NCCL has no "sum mod l" reduction anyway.
//   * bulk hand-overs (the per-rank partial points of a row-MSM, "bucket-sum reduce" = gather-then-add: group
//     addition is not an NCCL reduction either; the heads of the polynomials when one element per rank is left;
//     the LZ vector of an opening): an all-gather written here as ONE kernel that stores the rank's block into
//     every peer's exchange buffer over NVLink / NVSwitch peer memory (CUDA IPC), fences at system scope and
//     publishes a tagged completion marker to every process; the hosts wait for the G markers and the consumers
//     read their local exchange buffer.  Double-buffered by message parity: a peer can be at most one message
//     ahead, because its next push is stream-ordered after its own consumption of the current one.
//     LASSO_B200_XCHG=nccl selects ncclAllGather for these instead (the baseline this replaces; NCCL is loaded
//     with dlopen so the library has no link-time dependency on it).
// Because nothing here needs one DEVICE per rank, two ranks can share a GPU: the sharded path is exercised by
// the single-GPU test box too (tests/test_gpu_sharded.py).
#include <dlfcn.h>
#include <fcntl.h>
#include <nccl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include "prover.cuh"

namespace lb {

// ------------------------------------------------------------------------------------------ NCCL (optional)
struct NcclApi {
  void* h = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
};
static NcclApi& nccl() {
  static NcclApi api;
  if (!api.h) {
    const char* names[] = {getenv("LASSO_B200_NCCL"), "libnccl.so.2", "libnccl.so"};
    for (const char* n : names) {
      if (!n) continue;
      api.h = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
      if (api.h) break;
    }
    if (!api.h) throw std::runtime_error("cannot dlopen libnccl.so.2 (set LASSO_B200_NCCL)");
    api.GetUniqueId = (decltype(api.GetUniqueId))dlsym(api.h, "ncclGetUniqueId");
    api.CommInitRank = (decltype(api.CommInitRank))dlsym(api.h, "ncclCommInitRank");
    api.CommDestroy = (decltype(api.CommDestroy))dlsym(api.h, "ncclCommDestroy");
    api.AllGather = (decltype(api.AllGather))dlsym(api.h, "ncclAllGather");
    api.GetErrorString = (decltype(api.GetErrorString))dlsym(api.h, "ncclGetErrorString");
    if (!api.GetUniqueId || !api.CommInitRank || !api.AllGather) throw std::runtime_error("libnccl: missing symbols");
  }
  return api;
}
#define LB_NCCL_CHECK(x)                                                                        \
  do {                                                                                          \
    ncclResult_t r_ = (x);                                                                      \
    if (r_ != ncclSuccess)                                                                      \
      throw std::runtime_error(std::string("NCCL error: ") + nccl().GetErrorString(r_));        \
  } while (0)
static bool want_nccl() {
  const char* m = getenv("LASSO_B200_XCHG");
  return m && std::string(m) == "nccl";
}

// ------------------------------------------------------------------------------------------ shared segments
static constexpr size_t kSegHeaderBytes = 4096;
static constexpr size_t kXchgSlotBytes = (size_t)2 << 20;  // per (parity, writer)
struct SegHeader {  // the first bytes of a rank's shared host segment (zero-filled at creation)
  volatile uint64_t ready;                    // 1: the fields below are valid
  volatile uint64_t opened[kPubMaxReaders];   // opened[w]: rank w has mapped this segment and imported the buffer
  volatile uint64_t closed[kPubMaxReaders];   // closed[w]: rank w has released its import again
  uint64_t has_ipc;
  cudaIpcMemHandle_t xbuf_handle;             // the rank's device exchange buffer
};
static_assert(sizeof(SegHeader) <= kSegHeaderBytes, "segment header");

struct Xchg {
  int world = 1, rank = 0;
  size_t seg_bytes = 0;
  std::string name[kPubMaxReaders];
  void* seg[kPubMaxReaders] = {};      // host mappings of every rank's segment (own included)
  bool registered[kPubMaxReaders] = {};
  uint8_t* xbuf[kPubMaxReaders] = {};  // device: every rank's exchange buffer ([rank] = own allocation)
  uint32_t xseq = 0;
  ncclComm_t nccl_comm = nullptr;  // LASSO_B200_XCHG=nccl
};
static Xchg* xc(Ctx* c) { return (Xchg*)c->xchg; }

static uint64_t fnv64(const uint8_t* p, size_t n) {
  uint64_t h = 1469598103934665603ull;
  for (size_t i = 0; i < n; i++) h = (h ^ p[i]) * 1099511628211ull;
  return h;
}
template <class F>
static void wait_until(F cond, double seconds, const char* what) {
  auto t0 = std::chrono::steady_clock::now();
  while (!cond()) {
    usleep(200);
    if (std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count() > seconds)
      throw std::runtime_error(std::string("timeout waiting for the other ranks: ") + what);
  }
}

void comm_unique_id(uint8_t out[128]) {
  if (want_nccl()) {
    ncclUniqueId id;
    LB_NCCL_CHECK(nccl().GetUniqueId(&id));
    static_assert(sizeof(id) == 128, "ncclUniqueId size");
    memcpy(out, &id, 128);
    return;
  }
  // the id only names the job's shared segments: 128 random bytes
  int fd = open("/dev/urandom", O_RDONLY);
  if (fd < 0 || read(fd, out, 128) != 128) {
    if (fd >= 0) close(fd);
    throw std::runtime_error("cannot read /dev/urandom");
  }
  close(fd);
}

// undo whatever of a (partially) built exchange exists: imports, registrations, mappings, the own buffer and name
static void xchg_release(Xchg* x) {
  if (!x) return;
  if (x->nccl_comm) nccl().CommDestroy(x->nccl_comm);
  x->nccl_comm = nullptr;
  for (int r = 0; r < x->world; r++) {
    if (r != x->rank && x->xbuf[r]) cudaIpcCloseMemHandle(x->xbuf[r]);
    if (r != x->rank) x->xbuf[r] = nullptr;
  }
  for (int r = 0; r < x->world; r++) {
    if (x->registered[r]) cudaHostUnregister(x->seg[r]);
    x->registered[r] = false;
    if (x->seg[r]) munmap(x->seg[r], x->seg_bytes);
    x->seg[r] = nullptr;
  }
  if (x->xbuf[x->rank]) cudaFree(x->xbuf[x->rank]);
  x->xbuf[x->rank] = nullptr;
  if (!x->name[x->rank].empty()) shm_unlink(x->name[x->rank].c_str());  // harmless if it is gone already
}

static void comm_init_impl(Ctx* c, Xchg* x, const uint8_t id_bytes[128], int rank, int world);
void comm_init(Ctx* c, const uint8_t id_bytes[128], int rank, int world) {
  if (world < 1 || (world & (world - 1)) || world > kPubMaxReaders || rank < 0 || rank >= world)
    throw std::runtime_error("world must be a power of two <= 8 (one node)");
  if (c->xchg) throw std::runtime_error("communicator already initialised");
  LB_CUDA_CHECK(cudaSetDevice(c->device));
  c->world = world;
  c->rank = rank;
  c->lg_world = 0;
  while ((1 << c->lg_world) < world) c->lg_world++;
  if (world == 1) return;
  std::unique_ptr<Xchg> x(new Xchg());
  try {
    comm_init_impl(c, x.get(), id_bytes, rank, world);
  } catch (...) {  // a failed or timed-out rendezvous must not leave mappings, registrations or a shm name behind
    xchg_release(x.get());
    if (c->d_gather) cudaFree(c->d_gather);
    c->d_gather = nullptr;
    c->world = 1;
    c->rank = 0;
    c->lg_world = 0;
    throw;
  }
  c->xchg = x.release();
}
static void comm_init_impl(Ctx* c, Xchg* x, const uint8_t id_bytes[128], int rank, int world) {
  x->world = world;
  x->rank = rank;
  x->seg_bytes = kSegHeaderBytes + Ctx::kPubBytes;
  const uint64_t job = fnv64(id_bytes, 128);
  for (int r = 0; r < world; r++) {
    char nm[96];
    snprintf(nm, sizeof nm, "/lasso_b200_%016llx_%d", (unsigned long long)job, r);
    x->name[r] = nm;
  }
  // own exchange buffer + own segment
  const size_t xbytes = 2 * (size_t)kPubMaxReaders * kXchgSlotBytes;
  LB_CUDA_CHECK(cudaMalloc((void**)&x->xbuf[rank], xbytes));
  LB_CUDA_CHECK(cudaMemset(x->xbuf[rank], 0, xbytes));
  {
    shm_unlink(x->name[rank].c_str());
    int fd = shm_open(x->name[rank].c_str(), O_CREAT | O_EXCL | O_RDWR, 0600);
    if (fd < 0) throw std::runtime_error("shm_open(create) failed for " + x->name[rank]);
    if (ftruncate(fd, (off_t)x->seg_bytes) != 0) {
      close(fd);
      throw std::runtime_error("ftruncate failed on the shared segment");
    }
    void* p = mmap(nullptr, x->seg_bytes, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
    close(fd);
    if (p == MAP_FAILED) throw std::runtime_error("mmap failed on the shared segment");
    memset(p, 0, x->seg_bytes);
    x->seg[rank] = p;
    LB_CUDA_CHECK(cudaHostRegister(p, x->seg_bytes, cudaHostRegisterMapped | cudaHostRegisterPortable));
    x->registered[rank] = true;
    SegHeader* h = (SegHeader*)p;
    if (!want_nccl()) {
      LB_CUDA_CHECK(cudaIpcGetMemHandle(&h->xbuf_handle, x->xbuf[rank]));
      h->has_ipc = 1;
    }
    __sync_synchronize();
    h->ready = 1;
  }
  // the other ranks' segments and exchange buffers
  for (int r = 0; r < world; r++) {
    if (r == rank) continue;
    int fd = -1;
    wait_until(
        [&] {
          fd = shm_open(x->name[r].c_str(), O_RDWR, 0600);
          if (fd < 0) return false;
          struct stat st;
          if (fstat(fd, &st) != 0 || (size_t)st.st_size < x->seg_bytes) {
            close(fd);
            fd = -1;
            return false;
          }
          return true;
        },
        120.0, "shared segment not created");
    void* p = mmap(nullptr, x->seg_bytes, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
    close(fd);
    if (p == MAP_FAILED) throw std::runtime_error("mmap failed on a peer's shared segment");
    x->seg[r] = p;
    SegHeader* h = (SegHeader*)p;
    wait_until([&] { return h->ready == 1; }, 120.0, "shared segment not ready");
    __sync_synchronize();
    LB_CUDA_CHECK(cudaHostRegister(p, x->seg_bytes, cudaHostRegisterMapped | cudaHostRegisterPortable));
    x->registered[r] = true;
    if (!want_nccl()) {
      if (!h->has_ipc) throw std::runtime_error("the ranks disagree on LASSO_B200_XCHG");
      cudaError_t e = cudaIpcOpenMemHandle((void**)&x->xbuf[r], h->xbuf_handle, cudaIpcMemLazyEnablePeerAccess);
      if (e != cudaSuccess)
        throw std::runtime_error(std::string("cudaIpcOpenMemHandle failed (") + cudaGetErrorString(e) +
                                 "): no peer access between the GPUs of this job; LASSO_B200_XCHG=nccl selects NCCL for the bulk exchanges");
    }
    h->opened[rank] = 1;
  }
  {
    SegHeader* h = (SegHeader*)x->seg[rank];
    wait_until(
        [&] {
          for (int r = 0; r < world; r++)
            if (r != rank && h->opened[r] != 1) return false;
          return true;
        },
        120.0, "peers did not map this rank's segment");
    shm_unlink(x->name[rank].c_str());  // every rank holds a mapping now: the name can go
  }
  if (want_nccl()) {
    ncclUniqueId id;
    memcpy(&id, id_bytes, 128);
    LB_NCCL_CHECK(nccl().CommInitRank(&x->nccl_comm, world, id, rank));
  }
  c->gather_elems = 1 << 16;
  LB_CUDA_CHECK(cudaMalloc((void**)&c->d_gather, c->gather_elems * sizeof(fr_t)));
  unsigned long long* readers[kPubMaxReaders] = {};
  for (int r = 0; r < world; r++) {
    void* dp = nullptr;
    LB_CUDA_CHECK(cudaHostGetDevicePointer(&dp, x->seg[r], 0));
    readers[r] = (unsigned long long*)((uint8_t*)dp + kSegHeaderBytes);
  }
  // publication: this process now receives in its shared segment and sees every reader's segment.  Nothing below
  // can fail: a failed initialisation leaves the context with its own publication buffer.
  if (c->h_pub_owned) cudaFreeHost(c->h_pub);
  c->h_pub_owned = false;
  c->h_pub = (unsigned long long*)((uint8_t*)x->seg[rank] + kSegHeaderBytes);
  for (int r = 0; r < world; r++) c->d_pub_reader[r] = readers[r];
  c->pub_seq = 0;
  c->pub_ring[0] = c->pub_ring[1] = 0;
}

void comm_destroy(Ctx* c) {
  Xchg* x = xc(c);
  if (!x) return;
  cudaSetDevice(c->device);
  cudaStreamSynchronize(c->st);
  if (x->nccl_comm) nccl().CommDestroy(x->nccl_comm);
  for (int r = 0; r < x->world; r++) {
    if (r == x->rank) continue;
    if (x->xbuf[r]) cudaIpcCloseMemHandle(x->xbuf[r]);
    if (x->seg[r]) ((SegHeader*)x->seg[r])->closed[x->rank] = 1;
  }
  if (x->seg[x->rank]) {  // do not free what a peer may still have imported (bounded wait: a dead peer must not hang us)
    SegHeader* h = (SegHeader*)x->seg[x->rank];
    auto t0 = std::chrono::steady_clock::now();
    for (;;) {
      bool all = true;
      for (int r = 0; r < x->world; r++)
        if (r != x->rank && h->opened[r] == 1 && h->closed[r] != 1) all = false;
      if (all || std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count() > 10.0) break;
      usleep(200);
    }
  }
  for (int r = 0; r < x->world; r++) {
    if (x->registered[r]) cudaHostUnregister(x->seg[r]);
    if (x->seg[r]) munmap(x->seg[r], x->seg_bytes);
  }
  if (x->xbuf[x->rank]) cudaFree(x->xbuf[x->rank]);
  if (c->d_gather) cudaFree(c->d_gather);
  c->d_gather = nullptr;
  c->h_pub = nullptr;  // it lived in the segment
  for (int r = 0; r < kPubMaxReaders; r++) c->d_pub_reader[r] = nullptr;
  c->xchg = nullptr;
  c->world = 1;
  c->rank = 0;
  c->lg_world = 0;
  delete x;
}

// ------------------------------------------------------------------------------------------ all-gather
struct PeerPtrs {
  uint4* p[kPubMaxReaders];
};
// Every rank runs this with its own block: the block is stored into slot `rank` of EVERY peer's exchange buffer
// (P2P stores over NVLink; the own buffer is one of the destinations), then the last CTA — after every thread's
// system-scope fence — publishes the completion marker to every process.
__global__ void __launch_bounds__(256)
    xchg_push_kernel(const uint4* src, size_t n16, PeerPtrs peers, int world, unsigned* counter, PubDst marker, uint32_t seq) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += (size_t)gridDim.x * blockDim.x) {
    const uint4 v = src[i];
    for (int p = 0; p < world; p++) peers.p[p][i] = v;
  }
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();
    if (atomicAdd(counter, 1u) == gridDim.x - 1) {
      *counter = 0;
      __threadfence_system();
      uint32_t one[8] = {seq, 0, 0, 0, 0, 0, 0, 0};
      pub_store(marker, 0, one);
    }
  }
}
// recv[g * bytes_per_rank ..) = rank g's send buffer, on every rank
void comm_allgather(Ctx* c, const void* d_send, void* d_recv, size_t bytes_per_rank) {
  if (c->world == 1) {
    if (d_send != d_recv) LB_CUDA_CHECK(cudaMemcpyAsync(d_recv, d_send, bytes_per_rank, cudaMemcpyDeviceToDevice, c->st));
    return;
  }
  Xchg* x = xc(c);
  if (x->nccl_comm) {
    LB_NCCL_CHECK(nccl().AllGather(d_send, d_recv, bytes_per_rank, ncclChar, x->nccl_comm, c->st));
    return;
  }
  if (bytes_per_rank % 16) throw std::runtime_error("allgather: block size must be a multiple of 16 bytes");
  for (size_t off = 0; off < bytes_per_rank; off += kXchgSlotBytes) {
    const size_t chunk = std::min(kXchgSlotBytes, bytes_per_rank - off);
    const uint32_t seq = ++x->xseq;
    const size_t par = seq & 1;
    PeerPtrs peers;
    for (int r = 0; r < c->world; r++) peers.p[r] = (uint4*)(x->xbuf[r] + (par * kPubMaxReaders + c->rank) * kXchgSlotBytes);
    const PubDst marker = c->pub_begin(true);
    const size_t n16 = chunk / 16;
    unsigned blocks = (unsigned)std::min<size_t>((n16 + 255) / 256, (size_t)kNumSMs);
    if (blocks < 1) blocks = 1;
    launch(xchg_push_kernel, blocks, 256, 0, c->st, (const uint4*)((const uint8_t*)d_send + off), n16, peers, c->world,
           c->d_flag + 8, marker, seq);
    uint32_t got[8];
    for (int w = 0; w < c->world; w++) c->pub_wait_raw(marker, w, 1, got);  // every rank's block has landed here
    LB_CUDA_CHECK(cudaMemcpy2DAsync((uint8_t*)d_recv + off, bytes_per_rank, x->xbuf[c->rank] + par * kPubMaxReaders * kXchgSlotBytes,
                                    kXchgSlotBytes, chunk, (size_t)c->world, cudaMemcpyDeviceToDevice, c->st));
  }
}

// tail hand-over: every rank holds ONE element of each of npolys polynomials (local length 1), optionally one
// more (`extra`, the shared eq polynomial of a grand-product layer) as polynomial number npolys;
// afterwards out[k*G + g] = rank g's element of polynomial k, on every rank (global index = g).
__global__ void pack_heads_kernel(fr_t* const* ptrs, const fr_t* base, size_t stride, int npolys, const fr_t* extra, fr_t* out) {
  int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < npolys) out[k] = ptrs ? ptrs[k][0] : base[(size_t)k * stride];
  if (k == npolys && extra) out[k] = extra[0];
}
__global__ void transpose_gathered_kernel(const fr_t* gathered /*[G][npolys]*/, int world, int npolys, fr_t* out /*[npolys][G]*/) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= world * npolys) return;
  int g = i / npolys, k = i % npolys;
  out[(size_t)k * world + g] = gathered[i];
}
// out[k] = ptrs[k][0] (or base[k*stride]): used to bring the 2*ncirc final claims of a layer to the host in one go
void pack_heads(Ctx* c, fr_t* const* d_ptrs, const fr_t* base, size_t stride, int npolys, fr_t* d_out) {
  launch(pack_heads_kernel, (npolys + 127) / 128, 128, 0, c->st, d_ptrs, base, stride, npolys, nullptr, d_out);
}
void comm_gather_heads(Ctx* c, fr_t* const* d_ptrs, const fr_t* base, size_t stride, int npolys, const fr_t* extra, fr_t* d_out) {
  const int total = npolys + (extra ? 1 : 0);
  if ((size_t)total * (c->world + 1) > c->gather_elems) throw std::runtime_error("gather_heads: too many polynomials");
  fr_t* packed = c->d_gather + (size_t)total * c->world;
  launch(pack_heads_kernel, (total + 127) / 128, 128, 0, c->st, d_ptrs, base, stride, npolys, extra, packed);
  comm_allgather(c, packed, c->d_gather, (size_t)total * sizeof(fr_t));
  launch(transpose_gathered_kernel, (total * c->world + 127) / 128, 128, 0, c->st, c->d_gather, c->world, total, d_out);
}
// in[g * n_loc + j] (rank g's block of n_loc elements) -> out[j * G + g]: the low-bit shards of a vector, interleaved
__global__ void __launch_bounds__(256) interleave_kernel(const fr_t* in, int world, size_t n_loc, fr_t* out) {
  const size_t n = n_loc * world;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const size_t g = i / n_loc, j = i - g * n_loc;
    st_fr(out + j * world + g, ld_fr(in + i));
  }
}
// every rank holds the low-bit shard (n_loc elements) of a vector; d_out receives the whole vector on every rank
void comm_gather_vector(Ctx* c, const fr_t* d_shard, size_t n_loc, fr_t* d_scratch /* n_loc * G */, fr_t* d_out) {
  if (c->world == 1) {
    if (d_out != d_shard) LB_CUDA_CHECK(cudaMemcpyAsync(d_out, d_shard, n_loc * sizeof(fr_t), cudaMemcpyDeviceToDevice, c->st));
    return;
  }
  comm_allgather(c, d_shard, d_scratch, n_loc * sizeof(fr_t));
  const size_t n = n_loc * c->world;
  launch(interleave_kernel, (unsigned)std::min<size_t>((n + 255) / 256, 4 * (size_t)kNumSMs), 256, 0, c->st, d_scratch,
         c->world, n_loc, d_out);
}

}  // namespace lb
