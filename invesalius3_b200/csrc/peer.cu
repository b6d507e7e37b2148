// Peer mailboxes over NVLink (cudaIpc): allocation, export, mapping. See peer.cuh for the
// layout and the protocol. The reference has no multi-GPU code at all; its only decomposition
// is the Z-piece split of surface extraction through temp files
// (invesalius/data/surface.py:1360-1430) — these mailboxes replace that exchange.
#include <string.h>

#include "peer.cuh"

extern "C" int64_t b2v_peer_mailbox_bytes(int64_t dy, int64_t dx) {
  if (dy <= 0 || dx <= 0) return 0;
  return peer_mailbox_bytes(dy * ceil_div64(dx, 32) * 4);
}

extern "C" int b2v_peer_alloc(int64_t bytes, void** dev_ptr_out, uint8_t* handle_out /*[64]*/) {
  B2V_REQUIRE(bytes > 0 && dev_ptr_out && handle_out, B2V_ERR_ARG, "peer_alloc: bad arguments");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
  void* p = nullptr;
  B2V_CUDA(cudaMalloc(&p, (size_t)bytes));
  B2V_CUDA(cudaMemset(p, 0, (size_t)bytes));
  cudaIpcMemHandle_t h;
  cudaError_t e = cudaIpcGetMemHandle(&h, p);
  if (e != cudaSuccess) {
    cudaFree(p);
    b2v_set_error("cudaIpcGetMemHandle failed: %s", cudaGetErrorString(e));
    return B2V_ERR_CUDA;
  }
  B2V_CUDA(cudaDeviceSynchronize());
  memcpy(handle_out, &h, 64);
  *dev_ptr_out = p;
  return B2V_OK;
}

extern "C" int b2v_peer_open(const uint8_t* handle /*[64]*/, void** dev_ptr_out) {
  B2V_REQUIRE(handle && dev_ptr_out, B2V_ERR_ARG, "peer_open: bad arguments");
  cudaIpcMemHandle_t h;
  memcpy(&h, handle, 64);
  void* p = nullptr;
  B2V_CUDA(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
  *dev_ptr_out = p;
  return B2V_OK;
}

extern "C" int b2v_peer_close(void* mapped_ptr) {
  if (!mapped_ptr) return B2V_OK;
  B2V_CUDA(cudaIpcCloseMemHandle(mapped_ptr));
  return B2V_OK;
}

extern "C" int b2v_peer_free(void* dev_ptr) {
  if (!dev_ptr) return B2V_OK;
  B2V_CUDA(cudaFree(dev_ptr));
  return B2V_OK;
}

int peer_make_set(int rank, int world, const void* const* mailboxes_host, int64_t plane_bytes, uint32_t epoch,
                  PeerSet* out) {
  B2V_REQUIRE(world >= 1 && world <= kPeerMaxWorld && rank >= 0 && rank < world && mailboxes_host && plane_bytes > 0,
              B2V_ERR_ARG, "peer: bad rank / world (at most %d ranks) / mailboxes", kPeerMaxWorld);
  memset(out, 0, sizeof(*out));
  out->rank = rank;
  out->world = world;
  out->epoch = epoch;
  out->pc = plane_bytes;
  // ~4 s of SM clocks. The clock-rate attribute is one of the slow driver queries:
  // asked once per process, not per call.
  static long long cached_timeout = 0;
  if (cached_timeout == 0) {
    int dev = 0, khz = 0;
    B2V_CUDA(cudaGetDevice(&dev));
    if (cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, dev) != cudaSuccess || khz <= 0) khz = 1500000;
    cached_timeout = (long long)khz * 1000ll * 4ll;
  }
  out->timeout = cached_timeout;
  for (int r = 0; r < world; ++r) {
    B2V_REQUIRE(mailboxes_host[r], B2V_ERR_ARG, "peer: mailbox of rank %d is not mapped", r);
    out->box[r] = (char*)const_cast<void*>(mailboxes_host[r]);
  }
  return B2V_OK;
}

// ---- a barrier over the mailboxes (used by tests and as the self-check of a new link) -------------
// Every rank writes `epoch` into flags(parity)[rank] of every mailbox, then waits until its own
// mailbox holds `epoch` from everyone. ok_dev (device int) = 1 on success, 0 on timeout.
__global__ void k_peer_barrier(PeerSet ps, int* ok_dev) {
  const int t = threadIdx.x;
  const int parity = ps.epoch & 1;
  const uint32_t tag = ps.epoch * 2u;   // the flood kernel tags  epoch * 2 + changed
  if (t < ps.world) st_release_sys(ps.of(t).flags(parity) + ps.rank, tag);
  bool ok = true;
  if (t < ps.world) ok = peer_wait_eq(ps.mine().flags(parity) + t, tag, ps.timeout);
  ok = __syncthreads_and(ok);
  if (t == 0) *ok_dev = ok ? 1 : 0;
}

extern "C" int b2v_peer_barrier(int rank, int world, const void* const* mailboxes_host, int64_t plane_bytes,
                                uint32_t epoch, void* stream) {
  PeerSet ps;
  int rc = peer_make_set(rank, world, mailboxes_host, plane_bytes, epoch, &ps);
  if (rc) return rc;
  int* ok_dev = (int*)(ps.mine().base + 64 * 4 - 4);   // last signal word, unused otherwise
  k_peer_barrier<<<1, 32, 0, (cudaStream_t)stream>>>(ps, ok_dev);
  if ((rc = b2v_check_launch("k_peer_barrier"))) return rc;
  int ok = 0;
  B2V_CUDA(cudaMemcpyAsync(&ok, ok_dev, sizeof(int), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  B2V_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
  B2V_REQUIRE(ok == 1, B2V_ERR_NOCONV, "peer barrier timed out (epoch %u): a rank is missing or out of step", epoch);
  return B2V_OK;
}
