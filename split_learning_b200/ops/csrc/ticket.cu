// Device-side competing consumers (SURVEY §2.5, reference src/train/VGG16.py:40-53,143-154): every stage-(i+1) replica of a
// cluster `basic_get`s ONE shared queue, so whichever replica is free takes the next activation, and the gradient returns
// to the client named in the message's `trace`.  Here the queue is a ticket ring in exported device memory:
//
//   producer (after the pass that filled its outbox slot):   t = atom.add.sys(tail);  entry[t % R] = {origin, it, gseq, b};
//                                                            fence.sys; st.release.sys(entry.seq, t + 1)
//   consumer (any replica, before it enqueues a program):    t = head; t >= total -> "round drained"; t >= tail -> "empty";
//                                                            atom.cas.sys(head, t, t + 1); ld.acquire.sys(entry.seq) == t + 1;
//                                                            read the entry
//
// A ticket is claimed by exactly one replica (the atomic), in FIFO order, and names the origin (whose outbox slot holds the
// payload and whose gradient mailbox receives dX) — the reference's `trace[-1]`.  The claim result goes to mapped pinned
// host memory: the host picks the program (origin, slot) to enqueue, which is also how it learns that the round is drained.
#include "sm90.cuh"

namespace slb {

// ring words (u32): [0] tail  [1] head  [2] aborted  [3] reserved, then entries of 8 words:
//   {seq, origin, it, gseq, batch, 0, 0, 0}
constexpr int TK_HDR = 16;
constexpr int TK_ENTRY = 8;

__global__ void ticket_publish_kernel(uint32_t* ring, int ring_entries, uint32_t origin, uint32_t it, const uint32_t* gseq_ctr,
                                      uint32_t batch) {
  pdl_trigger();
  pdl_wait();                                                   // the pass that filled the outbox slot is complete and visible
  const uint32_t t = atomicAdd_system(ring + 0, 1u);
  uint32_t* e = ring + TK_HDR + static_cast<size_t>(t % ring_entries) * TK_ENTRY;
  e[1] = origin;
  e[2] = it;
  e[3] = gseq_ctr ? *gseq_ctr + 1u : 0u;                         // flag value the origin's backward pass will wait for
  e[4] = batch;
  __threadfence_system();
  st_release_sys(e + 0, t + 1u);
}

// out (mapped pinned host memory, 8 x u32): {status, ticket, origin, it, gseq, batch, 0, 0}
//   status 1 = claimed, 2 = drained (all `total` tickets handed out), 3 = timeout / aborted, 4 = nothing published yet
// The claim never parks on the device: a ticket is taken (CAS on head) only when tail says one has been allocated, so the
// only spin is the short window between a producer's atom.add on tail and its release of the entry.  "Nothing yet" goes
// back to the host, which polls — a long-lived spinner would occupy an SM slot and, on a GPU shared by many streams
// (several clients in one process), can sit in front of the very kernels that would publish the ticket it waits for.
__global__ void ticket_claim_kernel(uint32_t* ring, int ring_entries, uint32_t total, unsigned long long max_spins,
                                    volatile uint32_t* out) {
  pdl_wait();
  uint32_t t;
  for (;;) {
    t = ld_acquire_sys(ring + 1);
    if (t >= total) { out[1] = t; out[0] = 2u; __threadfence_system(); return; }
    if (t >= ld_acquire_sys(ring + 0)) { out[1] = t; out[0] = 4u; __threadfence_system(); return; }
    if (atomicCAS_system(ring + 1, t, t + 1u) == t) break;
  }
  out[1] = t;
  const uint32_t* e = ring + TK_HDR + static_cast<size_t>(t % ring_entries) * TK_ENTRY;
  unsigned long long spins = 0;
  while (ld_acquire_sys(e + 0) != t + 1u) {
    __nanosleep(100);
    if (++spins > max_spins || ld_acquire_sys(ring + 2) != 0u) { out[0] = 3u; __threadfence_system(); return; }
  }
  out[2] = e[1]; out[3] = e[2]; out[4] = e[3]; out[5] = e[4];
  __threadfence_system();
  out[0] = 1u;
  __threadfence_system();
}

__global__ void store_u32_kernel(uint32_t* p, uint32_t v) {
  pdl_trigger();
  pdl_wait();
  *p = v;
}

}  // namespace slb
using namespace slb;

extern "C" {

int slb_preload_ticket() {
  cudaFuncAttributes a;
  return (cudaFuncGetAttributes(&a, ticket_publish_kernel) != cudaSuccess) + (cudaFuncGetAttributes(&a, ticket_claim_kernel) != cudaSuccess) +
         (cudaFuncGetAttributes(&a, store_u32_kernel) != cudaSuccess);
}

int slb_ticket_ring_bytes(int ring_entries) { return (TK_HDR + ring_entries * TK_ENTRY) * 4; }

int slb_ticket_publish(uint32_t* ring, int ring_entries, uint32_t origin, uint32_t it, const uint32_t* gseq_ctr, uint32_t batch,
                       cudaStream_t st) {
  launch_k(ticket_publish_kernel, 1, 1, 0, st, ring, ring_entries, origin, it, gseq_ctr, batch);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : -static_cast<int>(e) - 2000;
}

int slb_ticket_claim(uint32_t* ring, int ring_entries, uint32_t total, unsigned long long max_spins, uint32_t* out_host,
                     cudaStream_t st) {
  uint32_t* dev_out = nullptr;
  if (cudaHostGetDevicePointer(reinterpret_cast<void**>(&dev_out), out_host, 0) != cudaSuccess) return -3;
  launch_k(ticket_claim_kernel, 1, 1, 0, st, ring, ring_entries, total, max_spins, dev_out);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : -static_cast<int>(e) - 2000;
}

int slb_store_u32(uint32_t* p, uint32_t v, cudaStream_t st) {
  launch_k(store_u32_kernel, 1, 1, 0, st, p, v);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : -static_cast<int>(e) - 2000;
}

}  // extern "C"
