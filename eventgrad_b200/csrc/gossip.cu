// eventgrad_b200 -- fused event-triggered gossip step (K1/K2) for sm_90a.
//
// What one launch does on every rank (persistent grid, one tile of EG_TILE floats per CTA
// iteration):
//   1. push   : tiles of tensors whose trigger fired are stored straight into the LEFT
//               neighbour's "from-right" inbox and the RIGHT neighbour's "from-left" inbox
//               (peer-mapped pointers -> NVLink 4 / NVSwitch).  Below threshold nothing is
//               stored, so link bytes scale with events (MPI_Put semantics,
//               /root/reference/dcifar10/event/event.cpp:317-332).
//   2. sync   : iter mode publishes one release-flag per (tile, warp) and waits for the two
//               neighbours' matching flags, so exchange and math overlap slice by slice;
//               async mode reads whatever the inboxes hold (reference: unsynchronised window
//               reads, event.cpp:372-374).
//   3. mix+opt: theta <- ((theta+L)+R)/3 ; m <- mu*m+g ; theta <- theta - lr*m   (event.cpp:
//               459-461, :479), rounding identical to add_/add_/div_/SGD.  Optionally with weight decay,
//               Nesterov momentum and a per-step learning rate read from a device table (sgd_elem/sched_lr,
//               common.cuh; off by default).
//   4. norm-on-write: per-warp sum theta_new^2 partials; the last CTA reduces them per tensor
//               in fixed order and runs the trigger FSM for the NEXT step (event.cpp:300-355),
//               so the step needs no extra pass over theta, no grid sync and no host sync.
//
// This file is compiled three times.  As gossip.cu it is the default kernel described above.  csrc/gossip_dbuf.cu
// defines EG_DBUF and includes it again to build the EXPERIMENTAL double-buffered dense variant
// (`gossip_step_kernel_dbuf`, decent only): the inbox has two slots, slot = step & 1, and the WAR ack
// (PROTOCOL.md 1.3) disappears -- a sender can be at most one step ahead of a receiver's reads because
// finishing step k+1 needs the receiver's flags of step k+1 (model-checked: tests/test_protocol_model.py).
// csrc/gossip_graph.cu defines EG_GRAPH and includes it a third time for circulant gossip graphs beyond the ring
// (`gossip_step_kernel_graph`, decent/event, fused step only): the two neighbours become the 2|O| inbox slots of a
// GraphSlots block that the graph kernel receives next to GossipParams (parallel/topology.py).  Each fired tile is
// pushed into every out-slot, iter mode publishes and waits for one flag per slot per (tile, warp), the tail acks
// every slot, and the mix adds the slots in slot order, two at a time, before one true division by 2|O|+1.
// With GraphSlots.period = tau > 0 the same kernel runs the time-varying one-peer exponential graph: at step k only slot
// m = (k-1) % tau is active (push into out-slot m, publish and wait on slot m's flags, ack slot m's sender, WAR guard on
// the ack of step k - tau) and the mix is (theta + in_m) / 2.  m comes from the device step counter (a uniform branch,
// no extra instance), so a captured launch replays every step of the cycle.
// GossipParams is unchanged, so the ring kernels compile exactly as before.
// Drift trigger (GossipParams.sent set, fsm.metric = 1): every fired tile that is pushed also stores theta_k into
// `sent` (the same thread that later mixes that tile, so no new cross-GPU ordering), and the norm-on-write partials
// become sum (theta_{k+1} - sent)^2, read after the SGD update once the gradient and momentum registers are dead.  The
// FSM then compares ||theta - sent|| with the threshold instead of | ||theta|| - ||theta at the last send|| |.
// csrc/gossip_q8.cu defines EG_Q8 and includes it a fourth time for int8 error-feedback compression of the ring's
// pushes (`gossip_step_kernel_q8`, decent/event, iter-sync fused step only): a fired tile's warp encodes theta - prev
// of its 256 elements as int8 codes plus one fp32 scale, stores them into the neighbours' code / scale inboxes of the
// Q8Slots block, and adds the dequantized delta to `prev`.  The (tile, warp) flag carries 2*step + fired, so the
// receiver learns from the flag whether to add the neighbour's delta to its replica before the mix
// ((theta + rep_l) + rep_r) / 3.  Under the drift trigger GossipParams.sent is `prev`.  Template parameters pick the
// codec (kSign: a 1-bit scaled sign per element, one byte per lane) and the mix (kChoco: CHOCO's
// theta + gamma * (((prev + rep_l) + rep_r) / 3 - prev)); Q8Slots.codec / gamma select the instance.
// csrc/gossip_gt.cu defines EG_GT and includes it a fifth time for gradient tracking (`gossip_step_kernel_gt`, decent
// on the ring, iter-sync fused step only): next to theta_k, the same thread pushes y_{k-1} of its slice into the
// neighbours' y inboxes of the TrackSlots block before the unchanged (tile, warp) flag, and the mix forms
// y_k = ((y + yL) + yR) / 3 + (g_k - g_prev) first, stores y and g_prev, mixes theta and hands y_k to sgd_elem in place
// of the gradient.  The ack of step k covers both inboxes, so there is no new synchronisation variable
// (PROTOCOL.md 1.8).
// csrc/gossip_ed.cu defines EG_ED and includes it a sixth time for exact diffusion (`gossip_step_kernel_ed`, decent on
// the ring, iter-sync fused step only; D^2 on W_bar = (I + W) / 2).  The optimizer moves from the mix to the push: the
// thread that owns a (tile, warp) slice runs p = sgd_elem(theta_k, g_k, ...) there, forms phi = p + (theta_k - psi),
// stores psi <- p, the momentum and phi into its own theta and both neighbours' inboxes, all before the unchanged flag.
// The mix then loads phi back (stored by the same thread), L and R and forms theta_{k+1} = (phi + ((phi + L) + R)/3) / 2
// with no optimizer.  Handshake, acks and the 2-rank single-copy dedup are the ring's (PROTOCOL.md 1.10).
// Periodic gossip (GossipParams.local_steps = H > 1, decent, ring and graph builds): step k pushes, flags, waits, mixes
// and acks only when H divides k; the other steps are the single-pass plain SGD step.  The WAR guard waits for the ack
// of the previous round (k - H; one-peer: k - tau * H) and the one-peer slot is indexed by the round k / H (PROTOCOL.md
// 1.9).
// Periodic global averaging (GossipParams.global_avg_period = P >= 2, decent, ring and static-graph builds): at step k
// with P dividing k, the gated all-reduce enqueued before this kernel (csrc/allreduce.cu, gate_period = P) has already
// replaced theta by the rank mean, and this kernel takes the same single-pass plain SGD step as a local step.  The
// other steps gossip; their WAR guard waits for the ack of the last step that gossiped (PROTOCOL.md 1.11).
// csrc/gossip_match.cu defines EG_MATCH and includes it a seventh time for random pairwise matchings
// (`gossip_step_kernel_match`, decent, iter-sync fused step only; --topology random-match): thread 0 of every CTA derives
// this step's partner from (seed, world, k) into shared memory (match_partner), the WAR guard waits for the partner's
// `done` word to reach k - 1, each warp pushes its slice into the partner's single inbox and publishes the (tile, warp)
// flag k there, waits for its own flag k and mixes (theta + inbox) / 2 as the one-peer graph does; the last CTA stores
// `done` = k.  An idle rank (odd world) takes the single-pass plain SGD step and still stores `done` (PROTOCOL.md 1.17).
// The int8, tracking and exact-diffusion builds derive their parameter block from GossipCore, which has no
// global_avg_period, so their slots keep their offsets; the launchers of every build but the ring and graph refuse P.
#include "api.h"
#include "common.cuh"
#include "sparse_apply.cuh"

namespace egb {
#ifdef EG_GRAPH
struct GraphStepParams : GossipParams {   // kernel parameter of the graph build: the ring block + the slots
  GraphSlots g;
};
using StepParams = GraphStepParams;
#elif defined(EG_Q8)
struct Q8StepParams : GossipCore {        // kernel parameter of the q8 build: the ring block + the int8 slots
  Q8Slots q;
};
using StepParams = Q8StepParams;
#elif defined(EG_GT)
struct GtStepParams : GossipCore {        // kernel parameter of the tracking build: the ring block + the y slots
  TrackSlots gt;
};
using StepParams = GtStepParams;
#elif defined(EG_ED)
struct EdStepParams : GossipCore {        // kernel parameter of the exact-diffusion build: the ring block + psi
  EdSlots ed;
};
using StepParams = EdStepParams;
#elif defined(EG_MATCH)
struct MatchStepParams : GossipParams {   // kernel parameter of the match build: the ring block + the matching
  MatchSlots m;
};
using StepParams = MatchStepParams;
#else
using StepParams = GossipParams;
#endif
}  // namespace egb

#if defined(EG_DBUF)
#define EG_SYM(name) name##_dbuf
#define EG_SLOT_OFF(p, step) ((size_t)((step) & 1) * ((size_t)(p).tab.n_tiles * EG_TILE))
#elif defined(EG_GRAPH)
#define EG_SYM(name) name##_graph
#define EG_SLOT_OFF(p, step) ((size_t)0)
#elif defined(EG_Q8)
#define EG_SYM(name) name##_q8
#define EG_SLOT_OFF(p, step) ((size_t)0)
#elif defined(EG_GT)
#define EG_SYM(name) name##_gt
#define EG_SLOT_OFF(p, step) ((size_t)0)
#elif defined(EG_ED)
#define EG_SYM(name) name##_ed
#define EG_SLOT_OFF(p, step) ((size_t)0)
#elif defined(EG_MATCH)
#define EG_SYM(name) name##_match
#define EG_SLOT_OFF(p, step) ((size_t)0)
#else
#define EG_SYM(name) name
#define EG_SLOT_OFF(p, step) ((size_t)0)
#endif
// messages one fired tensor costs: one per inbox slot it lands in (the reference's logical count)
#ifdef EG_GRAPH
#define EG_NMSG(p) ((p).g.period ? 1ull : (unsigned long long)(p).g.n_slots)
// one-peer graph: the slot of step `step` (1-based); static graphs and the ring have no active slot
#define EG_ACTIVE_SLOT(p, step) ((p).g.period ? ((step) - 1) % (p).g.period : -1)
#else
#define EG_NMSG(p) 2ull
#define EG_ACTIVE_SLOT(p, step) (-1)
#endif
// Periodic gossip (GossipParams.local_steps = H > 1) exists in the ring and graph builds only; the other builds gossip
// at every step and their launchers reject H > 1
#if defined(EG_DBUF) || defined(EG_Q8) || defined(EG_GT) || defined(EG_ED) || defined(EG_MATCH)
#define EG_LOCAL_STEPS 0
#else
#define EG_LOCAL_STEPS 1
#endif
// Quasi-global momentum (GossipParams.quasi_global) exists in the ring, double-buffered and graph builds; the int8,
// tracking and exact-diffusion builds take GossipCore, which has no such field, and their launchers reject it
#if defined(EG_Q8) || defined(EG_GT) || defined(EG_ED) || defined(EG_MATCH)
#define EG_QG 0
#else
#define EG_QG 1
#endif
#ifdef EG_GRAPH
static_assert(offsetof(egb::GraphStepParams, g) == sizeof(egb::GossipCore) + 8,
              "GraphSlots moved: quasi_global must stay in GossipParams' tail padding");
#endif

namespace egb {

#if EG_LOCAL_STEPS
// Is 1-based step `step` a global-averaging step (--global-avg-period P: iff P divides it)?  The launchers refuse P = 1
// and P < 0, so P > 0 means P >= 2
__device__ __forceinline__ bool global_avg_step(const StepParams& p, int step) {
  return p.global_avg_period > 0 && step % p.global_avg_period == 0;
}
#endif

// Does 1-based step `step` gossip?  --local-steps H: iff H divides it; --global-avg-period P: iff P does not divide it.
// Re-evaluated where it is needed instead of held in a register across the tile loops
__device__ __forceinline__ bool gossip_step_comm(const StepParams& p, int step) {
#if EG_LOCAL_STEPS
  return (p.local_steps <= 1 || step % p.local_steps == 0) && !global_avg_step(p, step);
#else
  return true;
#endif
}

// Per-CTA tile metadata, resolved ONCE at kernel start (thread j resolves iteration j, so the
// dependent table look-ups tile->tensor->{fire, grad pointer, numel} run in parallel instead of
// sitting on every iteration's critical path in front of the streaming loads).
struct TileInfo {
  const void* gptr;   // table mode: address of this tile's first gradient element (null: flat arena)
  int tensor;
  int valid;          // elements of the tensor left from this tile's start (>= EG_TILE: full tile)
  int flags;          // bit0 fire, bit1 gradient is bf16
};
#define EG_TI_CACHE 64

// -------------------------------------------------------------------------------------------
// Trigger FSM update of ONE tensor for step `next_step` (scalar code, one lane).
// Also accounts the messages of the step that just ran (fire[i] still holds that decision).
// -------------------------------------------------------------------------------------------
__device__ __forceinline__ void fsm_update_tensor(const FsmDev& f, const TableDev& tab, int i, float norm,
                                                  float lnorm, float rnorm, bool have_recv, int next_step,
                                                  bool count, unsigned long long nmsg) {
  const int sz = tab.n_tensors;
  float* row_next = nullptr;   // log row of the decision (step next_step)
  float* row_cur = nullptr;    // log row of the step that just ran (receive-side norms)
  if (f.log_ring != nullptr && f.log_cap > 0) {
    row_next = f.log_ring + (size_t)((next_step - 1) % f.log_cap) * sz * 5;
    if (next_step >= 2) row_cur = f.log_ring + (size_t)((next_step - 2) % f.log_cap) * sz * 5;
  }
  if (row_cur != nullptr && have_recv) {
    row_cur[i * 5 + 3] = lnorm;
    row_cur[i * 5 + 4] = rnorm;
  }
  f.cur_norm[i] = norm;
  if (!f.enabled) return;
  if (count && f.fire[i]) {   // +2 events per fired tensor, one per ring neighbour (event.cpp:319); graph: one per slot
    atomicAdd(f.counters + 0, nmsg);
    atomicAdd(f.counters + 1, nmsg * (unsigned long long)tab.t_msg_bytes[i]);
    atomicAdd(f.counters + 2, 1ull);
  }
  // drift: `norm` already is ||theta - sent||; norm rule: the reference's |norm - last_norm|
  const float value_diff = f.metric ? norm : fabsf(__fsub_rn(norm, f.last_norm[i]));
  const float iter_diff = __fsub_rn((float)next_step, f.last_iter[i]);
  float th = (f.thres_type == 1) ? __fmul_rn(f.thres[i], f.horizon) : f.constant;
  const bool fire = (value_diff >= th) || (next_step < f.initial_comm_passes);
  if (row_next != nullptr) {
    row_next[i * 5 + 0] = norm;
    row_next[i * 5 + 1] = th;
    row_next[i * 5 + 2] = fire ? 1.f : 0.f;
  }
  if (fire) {
    const int H = f.history;
    float* sl = f.slopes + (size_t)i * H;
    double avg = 0.0;
    for (int j = 0; j < H - 1; ++j) {
      sl[j] = sl[j + 1];
      avg += (double)sl[j];
    }
    sl[H - 1] = __fdiv_rn(value_diff, iter_diff);
    avg += (double)sl[H - 1];
    avg /= (double)H;
    if (f.thres_type == 1) th = (float)avg;
    f.last_norm[i] = norm;
    f.last_iter[i] = (float)next_step;
  }
  f.thres[i] = th;
  f.fire[i] = fire ? 1 : 0;
}

// Fixed-order reduction of the per-warp partials of one tensor by ONE warp: every lane owns a
// strided subsequence (float4 loads, 4 independent accumulators), then a shuffle tree.
__device__ __forceinline__ double reduce_partials(const float* part, int n4, int lane) {
  const float4* p4 = reinterpret_cast<const float4*>(part);
  double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0;
  int j = lane;
  for (; j + 96 < n4; j += 128) {
    const float4 x0 = __ldcg(p4 + j), x1 = __ldcg(p4 + j + 32), x2 = __ldcg(p4 + j + 64), x3 = __ldcg(p4 + j + 96);
    a0 += ((double)x0.x + (double)x0.y) + ((double)x0.z + (double)x0.w);
    a1 += ((double)x1.x + (double)x1.y) + ((double)x1.z + (double)x1.w);
    a2 += ((double)x2.x + (double)x2.y) + ((double)x2.z + (double)x2.w);
    a3 += ((double)x3.x + (double)x3.y) + ((double)x3.z + (double)x3.w);
  }
  for (; j < n4; j += 32) {
    const float4 x0 = __ldcg(p4 + j);
    a0 += ((double)x0.x + (double)x0.y) + ((double)x0.z + (double)x0.w);
  }
  return warp_sum_d((a0 + a1) + (a2 + a3));
}

// Norm reduction + trigger, spread over the grid with no serial tail and no per-tile fences:
// every CTA, once it has finished ALL its tiles, adds the number of tiles it contributed to each
// tensor's completion counter (one fence per CTA, <= tiles-per-CTA atomics).  The CTA whose add
// completes a tensor reduces that tensor's per-warp partials in fixed order (one warp per tensor)
// and runs the trigger FSM for it.  Tiles of a CTA ascend, so equal tensors are consecutive.
#define EG_MAX_OWN 1024   // >= number of parameter tensors (asserted host-side)
__device__ __forceinline__ void cta_finish_tensors(const StepParams& p, const TileInfo* s_ti, int next_step,
                                                   bool count, bool recv_ok) {
  __shared__ int s_own[EG_MAX_OWN];
  __shared__ int s_nown;
  const int b = blockIdx.x, G = gridDim.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  __syncthreads();                       // every warp of this CTA has stored its partials
  if (tid == 0) {
    __threadfence();
    int nown = 0, cur = -1, cnt = 0;
    int j = 0;
    for (int t = b; ; t += G, ++j) {
      const int i = (t < p.tab.n_tiles) ? ((s_ti != nullptr && j < EG_TI_CACHE) ? s_ti[j].tensor : p.tab.tile_tensor[t]) : -2;
      if (i != cur) {
        if (cur >= 0) {
          const unsigned prev = atomicAdd(p.tensor_done + cur, (unsigned)cnt);
          if (prev + (unsigned)cnt == (unsigned)p.tab.t_tile_count[cur] && nown < EG_MAX_OWN) s_own[nown++] = cur;
        }
        cur = i;
        cnt = 0;
      }
      if (i == -2) break;
      ++cnt;
    }
    s_nown = nown;
  }
  __syncthreads();
  const int nown = s_nown;
  if (nown == 0) return;
  __threadfence();
  const bool recv = recv_ok && (p.tile_ss_l != nullptr);
  for (int k = warp; k < nown; k += EG_WARPS) {
    const int i = s_own[k];
    const size_t off = (size_t)p.tab.t_tile_start[i] * EG_WARPS;
    const int n4 = p.tab.t_tile_count[i] * EG_WARPS / 4;
    const double ss = reduce_partials(p.tile_ss + off, n4, lane);
    double sl = 0.0, sr = 0.0;
    if (recv) {
      sl = reduce_partials(p.tile_ss_l + off, n4, lane);
      sr = reduce_partials(p.tile_ss_r + off, n4, lane);
    }
    if (lane == 0) {
      p.tensor_done[i] = 0u;
      fsm_update_tensor(p.fsm, p.tab, i, (float)sqrt(ss), (float)sqrt(sl), (float)sqrt(sr), recv, next_step, count,
                        EG_NMSG(p));
    }
  }
}

// -------------------------------------------------------------------------------------------
#ifdef EG_GRAPH
// Slot loops run over EG_MAX_SLOTS with constant indices (unrolled, predicated on slot_on), so every slot pointer
// is read straight from the kernel's parameter bank.
// Slot k takes part in this step: every slot of a static graph, only the active slot of a one-peer graph.
__device__ __forceinline__ bool slot_on(const StepParams& p, int k, int slot) {
  return p.g.period ? k == slot : k < p.g.n_slots;
}
__device__ __forceinline__ void push_tile(const StepParams& p, size_t base, const F8& th, int slot) {
#pragma unroll
  for (int k = 0; k < EG_MAX_SLOTS; ++k)
    if (slot_on(p, k, slot)) st_f8(p.g.push[k] + base, th);
  if (p.sent != nullptr) st_f8(p.sent + base, th);   // drift trigger: what the receivers now hold
}
#elif defined(EG_Q8)
__device__ __forceinline__ void st_u32x2(void* p, uint32_t lo, uint32_t hi) {
  asm volatile("st.global.v2.u32 [%0], {%1,%2};" ::"l"(p), "r"(lo), "r"(hi) : "memory");
}
__device__ __forceinline__ void ld_u32x2_cg(const void* p, uint32_t& lo, uint32_t& hi) {
  asm volatile("ld.global.cg.v2.u32 {%0,%1}, [%2];" : "=r"(lo), "=r"(hi) : "l"(p));
}
// One block = the 256 elements of this warp's slice of the tile (base >> 8 is its (tile, warp) index).  Encode
// d = theta - prev with one scale per block, push the 8 codes of this lane to both neighbours (one 8-byte store each),
// lane 0 pushes the scale, and prev += deq.  Bit for bit parallel/trigger.py q8_encode / q8_decode.
// kSign: the 1-bit scaled-sign codec (sign_encode / sign_decode), one byte per lane and neighbour at base >> 3.  Only
// this thread's first `nvalid` elements belong to the tensor: the padding after it decodes to 0 and stays 0 in prev.
template <bool kSign = false>
__device__ __forceinline__ void push_tile(const StepParams& p, size_t base, const F8& th, int /*slot*/,
                                          int nvalid = EG_VEC) {
  F8 pv = ld_f8(p.q.prev + base);
  if (kSign) {
    F8 d;
    float a = 0.f;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      d.v[e] = __fsub_rn(th.v[e], pv.v[e]);
      a = __fadd_rn(a, fabsf(d.v[e]));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a = __fadd_rn(a, __shfl_xor_sync(0xffffffffu, a, o));
    const float s = __fdiv_rn(a, 256.f);
    uint32_t bits = 0u;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const bool neg = d.v[e] < 0.f;
      bits |= (neg ? 1u : 0u) << e;
      if (e < nvalid) pv.v[e] = __fadd_rn(pv.v[e], neg ? -s : s);
    }
    p.q.q_to_l[base >> 3] = (int8_t)bits;
    p.q.q_to_r[base >> 3] = (int8_t)bits;
    if ((threadIdx.x & 31) == 0) {
      p.q.s_to_l[base >> 8] = s;
      p.q.s_to_r[base >> 8] = s;
    }
    st_f8(p.q.prev + base, pv);
    return;
  }
  F8 d;
  float a = 0.f;
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    d.v[e] = __fsub_rn(th.v[e], pv.v[e]);
    a = fmaxf(a, fabsf(d.v[e]));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) a = fmaxf(a, __shfl_xor_sync(0xffffffffu, a, o));
  const float s = __fdiv_rn(a, 127.f);
  uint32_t lo = 0u, hi = 0u;
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const float qf = (s == 0.f) ? 0.f : fminf(fmaxf(rintf(__fdiv_rn(d.v[e], s)), -127.f), 127.f);
    const uint32_t b = (uint32_t)((int)qf) & 0xffu;
    if (e < 4)
      lo |= b << (8 * e);
    else
      hi |= b << (8 * (e - 4));
    pv.v[e] = __fadd_rn(pv.v[e], __fmul_rn(qf, s));
  }
  st_u32x2(p.q.q_to_l + base, lo, hi);
  st_u32x2(p.q.q_to_r + base, lo, hi);
  if ((threadIdx.x & 31) == 0) {
    p.q.s_to_l[base >> 8] = s;
    p.q.s_to_r[base >> 8] = s;
  }
  st_f8(p.q.prev + base, pv);
}
// Receive side of one neighbour: when it fired this block, add its dequantized delta to my replica of its prev (the
// same fp32 add it applied to prev) and store the replica back; return theta + replica.  kSign: the sign codec's byte,
// added to the first `nvalid` elements only (the rest is the tensor's padding).
template <bool kSign = false>
__device__ __forceinline__ F8 q8_recv_add(float* rep, const int8_t* qin, const float* sin, size_t base, F8 th,
                                          bool fired, int nvalid = EG_VEC) {
  F8 r = ld_f8(rep + base);
  if (fired && kSign) {
    const uint32_t bits = (uint32_t)__ldcg(reinterpret_cast<const unsigned char*>(qin) + (base >> 3));
    const float s = __ldcg(sin + (base >> 8));
#pragma unroll
    for (int e = 0; e < 8; ++e)
      if (e < nvalid) r.v[e] = __fadd_rn(r.v[e], ((bits >> e) & 1u) ? -s : s);
    st_f8(rep + base, r);
  } else if (fired) {
    uint32_t lo, hi;
    ld_u32x2_cg(qin + base, lo, hi);
    const float s = __ldcg(sin + (base >> 8));
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int qv = (int)(int8_t)(((e < 4) ? lo >> (8 * e) : hi >> (8 * (e - 4))) & 0xffu);
      r.v[e] = __fadd_rn(r.v[e], __fmul_rn((float)qv, s));
    }
    st_f8(rep + base, r);
  }
#pragma unroll
  for (int e = 0; e < 8; ++e) th.v[e] = __fadd_rn(th.v[e], r.v[e]);
  return th;
}
// wait_ge that returns the flag value it saw.  In the q8 build a flag of step k is 2k + fired, and the WAR ack makes
// the value seen exactly 2k or 2k + 1 (PROTOCOL.md 1.7).
__device__ __forceinline__ uint32_t wait_ge_value(const uint32_t* flag, uint32_t want, int* status,
                                                  uint64_t timeout_ns) {
  const uint32_t v = ld_acquire_sys(flag);
  if (v >= want) return v;
  wait_ge(flag, want, status, timeout_ns);
  return ld_acquire_sys(flag);
}
#elif defined(EG_GT)
// theta_k and y_{k-1} of this thread's 8 elements to both neighbours, both before the (tile, warp) flag.  The thread
// that later mixes this slice overwrites y with y_k only after this load (program order), so no new ordering is needed.
// push_r == nullptr: 2-rank ring, one copy of each (y_to_r is null too)
__device__ __forceinline__ void push_tile(const StepParams& p, size_t base, const F8& th, int /*slot*/) {
  const F8 y = ld_f8(p.gt.y + base);
  st_f8(p.push_l + base, th);
  st_f8(p.gt.y_to_l + base, y);
  if (p.push_r != nullptr) {
    st_f8(p.push_r + base, th);
    st_f8(p.gt.y_to_r + base, y);
  }
}
#elif defined(EG_ED)
// phi of this thread's 8 elements to both neighbours (ed_push_stage forms it).  push_r == nullptr: 2-rank ring, one copy
__device__ __forceinline__ void push_tile(const StepParams& p, size_t base, const F8& phi, int /*slot*/) {
  st_f8(p.push_l + base, phi);
  if (p.push_r != nullptr) st_f8(p.push_r + base, phi);
}
#elif defined(EG_MATCH)
// theta_k of this thread's 8 elements into the single inbox of this step's partner `slot` (>= 0: the caller never pushes
// on an idle step)
__device__ __forceinline__ void push_tile(const StepParams& p, size_t base, const F8& th, int slot) {
  st_f8(p.m.peers[slot].inbox + base, th);
}
// Partner of this rank at 1-based step `step`, or -1 when it is idle (thread 0 only): splitmix64 from
// (seed << 32) ^ step, Fisher-Yates over `pi` from the identity, pairs (pi[0], pi[1]), (pi[2], pi[3]), ...  Bit for bit
// parallel/topology.py match_perm / match_partner
__device__ __noinline__ int match_partner(int seed, int R, int rank, int step, short* pi) {
  for (int i = 0; i < R; ++i) pi[i] = (short)i;
  uint64_t x = ((uint64_t)(uint32_t)seed << 32) ^ (uint64_t)(uint32_t)step;
  for (int i = R - 1; i >= 1; --i) {
    x += 0x9E3779B97F4A7C15ull;
    uint64_t z = x;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    z ^= z >> 31;
    const int j = (int)(z % (uint64_t)(i + 1));
    const short v = pi[i];
    pi[i] = pi[j];
    pi[j] = v;
  }
  int pos = 0;
  while (pi[pos] != rank) ++pos;
  if ((R & 1) && pos == R - 1) return -1;
  return pi[pos ^ 1];
}
#else
__device__ __forceinline__ void push_tile(const StepParams& p, size_t base, const F8& th, int /*slot*/) {
  // push_r == nullptr: 2-rank ring, the one neighbour is both left and right and reads the single copy twice
  st_f8(p.push_l + base, th);
  if (p.push_r != nullptr) st_f8(p.push_r + base, th);
#ifndef EG_DBUF
  if (p.sent != nullptr) st_f8(p.sent + base, th);   // drift trigger: what the receivers now hold (once, also at R = 2)
#endif
}
#endif
#ifdef EG_DBUF
__device__ __forceinline__ void push_tile_slot(const StepParams& p, size_t base, const F8& th, int step) {
  push_tile(p, EG_SLOT_OFF(p, step) + base, th, -1);
}
#endif

__device__ __forceinline__ TileInfo resolve_tile(const StepParams& p, int t) {
  TileInfo ti;
  const int i = p.tab.tile_tensor[t];
  const int first = (t - p.tab.t_tile_start[i]) * EG_TILE;
  ti.tensor = i;
  ti.valid = p.tab.t_numel[i] - first;
  ti.flags = p.fsm.fire[i] ? 1 : 0;
  ti.gptr = nullptr;
  if (p.t_grad_ptr != nullptr) {
    const bool bf = p.t_grad_bf16[i] != 0;
    ti.flags |= bf ? 2 : 0;
    ti.gptr = reinterpret_cast<const char*>(p.t_grad_ptr[i]) + (size_t)first * (bf ? 2 : 4);
  }
  return ti;
}

__device__ __forceinline__ void fill_tile_cache(const StepParams& p, TileInfo* s_ti) {
  const int j = threadIdx.x;
  if (j < EG_TI_CACHE) {
    const int t = blockIdx.x + j * gridDim.x;
    if (t < p.tab.n_tiles) s_ti[j] = resolve_tile(p, t);
  }
  __syncthreads();
}
__device__ __forceinline__ TileInfo tile_info(const StepParams& p, const TileInfo* s_ti, int j, int t) {
  return (j < EG_TI_CACHE) ? s_ti[j] : resolve_tile(p, t);
}

// Gradient of this thread's 8 elements.  Flat mode: the fp32 grad arena.  Table mode: autograd's
// own gradient tensors are read in place (bf16 or fp32, exactly numel elements each) -- no
// AccumulateGrad kernels, no grad arena traffic, no zeroing.
__device__ __forceinline__ F8 load_grad(const StepParams& p, const TileInfo& ti, size_t base, int tid) {
  if (ti.gptr == nullptr) return ld_f8(p.grad + base);
  const int off = tid * EG_VEC;
  F8 g;
  if (ti.flags & 2) {
    const __nv_bfloat16* gp = reinterpret_cast<const __nv_bfloat16*>(ti.gptr);
    if (off + EG_VEC <= ti.valid) {
      const uint4 u = *reinterpret_cast<const uint4*>(gp + off);
      const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = __bfloat1622float2(h[e]);
        g.v[2 * e] = f.x;
        g.v[2 * e + 1] = f.y;
      }
    } else {
#pragma unroll
      for (int e = 0; e < 8; ++e) g.v[e] = (off + e < ti.valid) ? __bfloat162float(gp[off + e]) : 0.f;
    }
  } else {
    const float* gp = reinterpret_cast<const float*>(ti.gptr);
    if (off + EG_VEC <= ti.valid) {
      const float4 a = *reinterpret_cast<const float4*>(gp + off), b = *reinterpret_cast<const float4*>(gp + off + 4);
      g.v[0] = a.x; g.v[1] = a.y; g.v[2] = a.z; g.v[3] = a.w;
      g.v[4] = b.x; g.v[5] = b.y; g.v[6] = b.z; g.v[7] = b.w;
    } else {
#pragma unroll
      for (int e = 0; e < 8; ++e) g.v[e] = (off + e < ti.valid) ? gp[off + e] : 0.f;
    }
  }
  return g;
}

#ifdef EG_ED
// Exact diffusion, push stage of one (tile, warp) slice, before its flag: t = theta_k - psi; p = sgd_elem(theta_k, g_k)
// with this step's lr; psi <- p and the momentum stored; flat mode zeroes the gradient; phi = p + t goes into my theta
// (the mix of this slice, run later by this thread, reads it back) and to both neighbours
template <bool kMom>
__device__ __forceinline__ void ed_push_stage(const StepParams& p, const TileInfo& ti, size_t base, int step) {
  F8 th, t;
  {
    th = ld_f8(p.theta + base);
    const F8 ps = ld_f8(p.ed.psi + base);
#pragma unroll
    for (int e = 0; e < 8; ++e) t.v[e] = __fsub_rn(th.v[e], ps.v[e]);
  }
  {
    const F8 g = load_grad(p, ti, base, threadIdx.x);
    F8 m;
    if (kMom) m = ld_f8(p.mom + base);
    const float lr = sched_lr(p.lr_table, p.lr_len, p.lr, step);
#pragma unroll
    for (int e = 0; e < 8; ++e) th.v[e] = sgd_elem<kMom>(th.v[e], g.v[e], m.v[e], lr, p.mu, p.wd, p.nesterov);
    if (kMom) st_f8(p.mom + base, m);
  }
  st_f8(p.ed.psi + base, th);
  if (p.zero_grad && ti.gptr == nullptr) {
    F8 z;
#pragma unroll
    for (int e = 0; e < 8; ++e) z.v[e] = 0.f;
    st_f8(p.grad + base, z);
  }
#pragma unroll
  for (int e = 0; e < 8; ++e) th.v[e] = __fadd_rn(th.v[e], t.v[e]);
  st_f8(p.theta + base, th);
  push_tile(p, base, th, -1);
}
#endif

// mix + SGD + norm-on-write for one tile. `th` already holds theta_k for this thread's 8 floats.  `mix`: p.do_mix of
// a gossip step, false on a local step of --local-steps (plain SGD); the q8 and tracking builds always mix.  kSign and
// kChoco exist in the q8 build only: the codec of the received deltas and the CHOCO mix (Q8Slots in api.h)
template <bool kMom, bool kQG, bool kSign = false, bool kChoco = false>
__device__ __forceinline__ void mix_tile(const StepParams& p, int t, const TileInfo& ti, size_t base, F8 th,
                                         int lane, int warp, int step, int slot, bool mix) {
#ifdef EG_GRAPH
  // no receive-norm logging on graphs (file_write is ring only); slots are loaded two at a time after the gradient
  // and momentum, which keeps the kernel at 64 registers whatever the degree
  constexpr bool logrecv = false;
  float ssl = 0.f, ssr = 0.f;
  F8 m;
  const F8 g = load_grad(p, ti, base, threadIdx.x);
  if (kMom) m = ld_f8(p.mom + base);
  if (mix && p.g.period) {
    // one-peer graph: theta <- (theta + in_slot) / 2
    const float* in = p.g.inbox[0];
#pragma unroll
    for (int s = 1; s < EG_MAX_SLOTS; ++s)
      if (s == slot) in = p.g.inbox[s];
    const F8 A = ld_f8_cg(in + base);
#pragma unroll
    for (int e = 0; e < 8; ++e) th.v[e] = __fdiv_rn(__fadd_rn(th.v[e], A.v[e]), 2.f);
  } else if (mix) {
#pragma unroll
    for (int s = 0; s < EG_MAX_SLOTS; s += 2) {
      if (s < p.g.n_slots) {
        const F8 A = ld_f8_cg(p.g.inbox[s] + base), B = ld_f8_cg(p.g.inbox[s + 1] + base);
#pragma unroll
        for (int e = 0; e < 8; ++e) th.v[e] = __fadd_rn(__fadd_rn(th.v[e], A.v[e]), B.v[e]);
      }
    }
    const float k = (float)(p.g.n_slots + 1);
#pragma unroll
    for (int e = 0; e < 8; ++e) th.v[e] = __fdiv_rn(th.v[e], k);
  }
#elif defined(EG_MATCH)
  // one-peer mix with this step's partner: theta <- (theta + inbox) / 2, loaded after the gradient and momentum as the
  // graph build stages its slots.  mix is false on an idle step
  constexpr bool logrecv = false;
  float ssl = 0.f, ssr = 0.f;
  F8 m;
  const F8 g = load_grad(p, ti, base, threadIdx.x);
  if (kMom) m = ld_f8(p.mom + base);
  if (mix) {
    const F8 A = ld_f8_cg(p.m.inbox + base);
#pragma unroll
    for (int e = 0; e < 8; ++e) th.v[e] = __fdiv_rn(__fadd_rn(th.v[e], A.v[e]), 2.f);
  }
#elif defined(EG_Q8)
  // `slot` carries the sides whose neighbour fired this block (bit 0 left, bit 1 right), read from the flags.  The
  // replicas are loaded one side at a time after the gradient and momentum, as the graph build stages its slots
  constexpr bool logrecv = false;
  float ssl = 0.f, ssr = 0.f;
  F8 m;
  const F8 g = load_grad(p, ti, base, threadIdx.x);
  if (kMom && !kChoco) m = ld_f8(p.mom + base);
  if (kChoco) {
    // CHOCO: t = ((prev + rep_l) + rep_r) / 3, theta <- theta + gamma * (t - prev).  prev (stored by this thread's push
    // of this slice earlier in the step, or unchanged when it did not fire) is read twice, and theta (not passed by the
    // caller) and the momentum only once the replicas are summed: staged like the int8 mix, this spills
    const int nv = ti.valid - (int)threadIdx.x * EG_VEC;
    F8 acc = ld_f8(p.q.prev + base);
    acc = q8_recv_add<kSign>(p.q.rep_l, p.q.q_from_l, p.q.s_from_l, base, acc, (slot & 1) != 0, nv);
    acc = q8_recv_add<kSign>(p.q.rep_r, p.q.q_from_r, p.q.s_from_r, base, acc, (slot & 2) != 0, nv);
    {
      const F8 pv = ld_f8(p.q.prev + base);
#pragma unroll
      for (int e = 0; e < 8; ++e) acc.v[e] = __fsub_rn(__fdiv_rn(acc.v[e], 3.0f), pv.v[e]);
    }
    th = ld_f8(p.theta + base);
    const float gamma = p.q.gamma;
#pragma unroll
    for (int e = 0; e < 8; ++e) th.v[e] = __fadd_rn(th.v[e], __fmul_rn(gamma, acc.v[e]));
    if (kMom) m = ld_f8(p.mom + base);
  } else {
    const int nv = kSign ? ti.valid - (int)threadIdx.x * EG_VEC : EG_VEC;
    th = q8_recv_add<kSign>(p.q.rep_l, p.q.q_from_l, p.q.s_from_l, base, th, (slot & 1) != 0, nv);
    th = q8_recv_add<kSign>(p.q.rep_r, p.q.q_from_r, p.q.s_from_r, base, th, (slot & 2) != 0, nv);
#pragma unroll
    for (int e = 0; e < 8; ++e) th.v[e] = __fdiv_rn(th.v[e], 3.0f);
  }
#elif defined(EG_GT)
  // staged so the gradient registers die before theta and its inboxes are loaded (the caller passes no theta): (1) g,
  // g_prev -> g - g_prev, g_prev <- g; y, yL, yR -> y_k, stored; (2) theta and its inboxes, mix; (3) sgd_elem on y_k
  // (held in `g`, the optimizer's input)
  constexpr bool logrecv = false;
  float ssl = 0.f, ssr = 0.f;
  F8 g, m;
  {
    const F8 gk = load_grad(p, ti, base, threadIdx.x);
    const F8 gp = ld_f8(p.gt.g_prev + base);
#pragma unroll
    for (int e = 0; e < 8; ++e) g.v[e] = __fsub_rn(gk.v[e], gp.v[e]);
    st_f8(p.gt.g_prev + base, gk);
  }
  {
    const F8 y = ld_f8(p.gt.y + base), yl = ld_f8_cg(p.gt.y_in_l + base), yr = ld_f8_cg(p.gt.y_in_r + base);
#pragma unroll
    for (int e = 0; e < 8; ++e)
      g.v[e] = __fadd_rn(__fdiv_rn(__fadd_rn(__fadd_rn(y.v[e], yl.v[e]), yr.v[e]), 3.0f), g.v[e]);
    st_f8(p.gt.y + base, g);
  }
  {
    th = ld_f8(p.theta + base);
    const F8 L = ld_f8_cg(p.inbox_l + base), R = ld_f8_cg(p.inbox_r + base);
#pragma unroll
    for (int e = 0; e < 8; ++e) th.v[e] = __fdiv_rn(__fadd_rn(__fadd_rn(th.v[e], L.v[e]), R.v[e]), 3.0f);
  }
  if (kMom) m = ld_f8(p.mom + base);
#elif defined(EG_ED)
  // load-only: phi (stored into theta by this thread's push stage), L and R; the optimizer already ran in the push
  constexpr bool logrecv = false;
  float ssl = 0.f, ssr = 0.f;
  {
    th = ld_f8(p.theta + base);
    const F8 L = ld_f8_cg(p.inbox_l + base), R = ld_f8_cg(p.inbox_r + base);
#pragma unroll
    for (int e = 0; e < 8; ++e)
      th.v[e] = __fdiv_rn(__fadd_rn(th.v[e], __fdiv_rn(__fadd_rn(__fadd_rn(th.v[e], L.v[e]), R.v[e]), 3.0f)), 2.f);
  }
#else
  const bool logrecv = (p.tile_ss_l != nullptr);
  float ssl = 0.f, ssr = 0.f;
  // issue every load of the tile before the first dependent FP op (5 x 32 B in flight per lane).  Quasi-global momentum
  // loads the inboxes after the gradient and momentum instead, as the graph build stages its slots: it re-reads theta_k
  // after the mix and would not fit in 64 registers otherwise
  constexpr bool qg = kMom && kQG;
  F8 L, R, m;
  if (mix && !qg) {
#ifdef EG_DBUF
    L = ld_f8_cg(p.inbox_l + EG_SLOT_OFF(p, step) + base);
    R = ld_f8_cg(p.inbox_r + EG_SLOT_OFF(p, step) + base);
#else
    L = ld_f8_cg(p.inbox_l + base);
    R = ld_f8_cg(p.inbox_r + base);
#endif
  }
  const F8 g = load_grad(p, ti, base, threadIdx.x);
  if (kMom) m = ld_f8(p.mom + base);
  if (mix) {
    if (qg) {
#ifdef EG_DBUF
      L = ld_f8_cg(p.inbox_l + EG_SLOT_OFF(p, step) + base);
      R = ld_f8_cg(p.inbox_r + EG_SLOT_OFF(p, step) + base);
#else
      L = ld_f8_cg(p.inbox_l + base);
      R = ld_f8_cg(p.inbox_r + base);
#endif
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      th.v[e] = __fdiv_rn(__fadd_rn(__fadd_rn(th.v[e], L.v[e]), R.v[e]), 3.0f);
      if (logrecv) {
        ssl = __fmaf_rn(L.v[e], L.v[e], ssl);
        ssr = __fmaf_rn(R.v[e], R.v[e], ssr);
      }
    }
  }
#endif
#ifdef EG_ED
  float ss = 0.f;
#pragma unroll
  for (int e = 0; e < 8; ++e) ss = __fmaf_rn(th.v[e], th.v[e], ss);
  st_f8(p.theta + base, th);
  if (p.shadow != nullptr) st_bf16x8(p.shadow + base, th);
#else
  // learning rate of this step, looked up per tile (an L1 hit) rather than held in a register across the loop
  const float lr = sched_lr(p.lr_table, p.lr_len, p.lr, step);
  float ss = 0.f;
#if EG_QG
  if (kMom && kQG) {
    // quasi-global momentum needs theta_k, which the mix has overwritten in `th` (the graph build accumulates the slots
    // into it).  This thread has not stored this slice of theta yet, and nothing else stores theta during the step (the
    // pipeline, the split step and the sparse prologue write only inboxes), so p.theta still holds theta_k
    const F8 tk = ld_f8(p.theta + base);
    const float c = __fsub_rn(1.f, p.mu);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      th.v[e] = qg_sgd_elem(__fsub_rn(tk.v[e], th.v[e]), th.v[e], g.v[e], m.v[e], lr, p.mu, c, p.wd, p.nesterov);
      ss = __fmaf_rn(th.v[e], th.v[e], ss);
    }
  } else
#endif
  {
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      th.v[e] = sgd_elem<kMom>(th.v[e], g.v[e], m.v[e], lr, p.mu, p.wd, p.nesterov);
      ss = __fmaf_rn(th.v[e], th.v[e], ss);
    }
  }
  if (kMom) st_f8(p.mom + base, m);
  st_f8(p.theta + base, th);
  if (p.shadow != nullptr) st_bf16x8(p.shadow + base, th);
  if (p.zero_grad && ti.gptr == nullptr) {
    F8 z;
#pragma unroll
    for (int e = 0; e < 8; ++e) z.v[e] = 0.f;
    st_f8(p.grad + base, z);
  }
#endif
#if !defined(EG_DBUF) && !defined(EG_GT) && !defined(EG_ED)
  if (p.sent != nullptr) {
    // drift trigger: sum (theta_{k+1} - sent)^2 replaces sum theta_{k+1}^2.  sent was stored by this thread's push of
    // this tile (or by the split step's push phase / the sparse compaction, both stream-ordered before this kernel)
    const F8 sv = ld_f8(p.sent + base);
    ss = 0.f;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float d = __fsub_rn(th.v[e], sv.v[e]);
      ss = __fmaf_rn(d, d, ss);
    }
  }
#endif
  ss = warp_sum(ss);
  if (logrecv) {
    ssl = warp_sum(ssl);
    ssr = warp_sum(ssr);
  }
  if (!p.need_norm) return;
  if (lane == 0) {
    p.tile_ss[(size_t)t * EG_WARPS + warp] = ss;
    if (logrecv) {
      p.tile_ss_l[(size_t)t * EG_WARPS + warp] = ssl;
      p.tile_ss_r[(size_t)t * EG_WARPS + warp] = ssr;
    }
  }
}

// Elect the last CTA of the grid; it acks and bumps the step counter (the trigger FSM itself is
// run per tensor by whichever warp completes that tensor, see cta_finish_tensors).  A local step of --local-steps
// read no inbox and acks nothing.
__device__ __forceinline__ void grid_tail(const StepParams& p, int step, int slot) {
  const bool comm = gossip_step_comm(p, step);
  __shared__ int s_last;
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const unsigned prev = atomicAdd(p.ticket, 1u);
    s_last = (prev == gridDim.x - 1) ? 1 : 0;
  }
  __syncthreads();
  if (!s_last) return;
  if (threadIdx.x == 0) {
    *p.ticket = 0u;
    *p.fsm.pass_num = step;
#if defined(EG_GRAPH)
    if (p.sync && p.send_ack && comm) {
      // every CTA of this rank has finished reading its inboxes for `step`: ack every active slot's sender
      fence_sys();
#pragma unroll
      for (int s = 0; s < EG_MAX_SLOTS; ++s)
        if (slot_on(p, s, slot)) st_release_sys(p.g.ack_to[s], (uint32_t)step);
    }
#elif defined(EG_MATCH)
    if (p.sync && p.send_ack) {
      // every CTA of this rank has finished reading its inbox for `step` (idle ranks too): the partners of later steps
      // may write it
      fence_sys();
      st_release_sys(p.m.done, (uint32_t)step);
    }
#elif !defined(EG_DBUF)
    if (p.sync && p.send_ack && comm) {
      // every CTA of this rank has finished reading its inboxes for `step`
      fence_sys();
      st_release_sys(p.ack_to_l, (uint32_t)step);
      st_release_sys(p.ack_to_r, (uint32_t)step);
    }
#endif
  }
}

// phase 1 of the split step: push only.  Depends on theta_k and the trigger decisions alone, so
// it is launched on a side stream at the START of step k and its NVLink traffic hides behind the
// forward/backward pass.  Publishes ONE "all pushed" flag per neighbour when every CTA is done.
__device__ __forceinline__ void push_phase(const StepParams& p, int step) {
  __shared__ int s_last;
  const int b = blockIdx.x, G = gridDim.x, tid = threadIdx.x;
  if (p.sync) {
    __shared__ int s_ok;
    if (tid == 0) {   // WAR guard: neighbours have consumed what I pushed at step-1
      bool ok = wait_ge(p.ack_from_l, (uint32_t)(step - 1), p.status, p.timeout_ns);
      ok = wait_ge(p.ack_from_r, (uint32_t)(step - 1), p.status, p.timeout_ns) && ok;
      s_ok = ok ? 1 : 0;
    }
    __syncthreads();
    if (!s_ok) return;   // a wedged / dead peer (sticky status set): never overwrite memory it may still be reading
  }
  __shared__ TileInfo s_ti[EG_TI_CACHE];
  fill_tile_cache(p, s_ti);
  int j = 0;
  for (int t = b; t < p.tab.n_tiles; t += G, ++j) {
    if (!(tile_info(p, s_ti, j, t).flags & 1)) continue;
    const size_t base = (size_t)t * EG_TILE + (size_t)tid * EG_VEC;
    push_tile(p, base, ld_f8(p.theta + base), -1);
  }
  __syncthreads();
  if (tid == 0) {
    __threadfence_system();
    const unsigned prev = atomicAdd(p.ticket + 1, 1u);
    s_last = (prev == gridDim.x - 1) ? 1 : 0;
  }
  __syncthreads();
  if (s_last && tid == 0) {
    p.ticket[1] = 0u;
    __threadfence_system();
    st_release_sys(p.pushed_to_l, (uint32_t)step);
    st_release_sys(p.pushed_to_r, (uint32_t)step);
  }
}

#if EG_QG
template <bool kMom, bool kQG>   // kQG: quasi-global momentum, an instance of its own (see DESIGN §4)
#elif defined(EG_Q8)
template <bool kMom, bool kSign, bool kChoco>   // kSign: the 1-bit sign codec; kChoco: the CHOCO mix (Q8Slots)
#else
template <bool kMom>
#endif
__global__ void __launch_bounds__(EG_THREADS, 4) EG_SYM(gossip_step_kernel)(const StepParams p) {
#if !EG_QG
  constexpr bool kQG = false;
#endif
  const int b = blockIdx.x, G = gridDim.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int step = *p.fsm.pass_num + 1;
  // --local-steps H: step k gossips iff H divides k, as round k / H; every other step is the serial SGD step.
  // --global-avg-period P: a step with P dividing k is the serial SGD step on the averaged theta.  A uniform branch on
  // the device pass counter, which iter-sync keeps equal on every rank (PROTOCOL.md 1.9, 1.11)
#ifdef EG_MATCH
  // this step's partner, -1 when idle (uniform per grid): an idle step is the single-pass plain SGD step
  __shared__ int s_partner;
  __shared__ short s_pi[EG_MATCH_MAX_WORLD];
  if (tid == 0) s_partner = match_partner(p.m.seed, p.m.world, p.m.rank, step, s_pi);
  __syncthreads();
  const int slot = s_partner;
  const bool comm = slot >= 0;
#else
  const bool comm = gossip_step_comm(p, step);
#if EG_LOCAL_STEPS
  const int H = max(p.local_steps, 1);
  const int slot = EG_ACTIVE_SLOT(p, step / H);
#else
  const int slot = EG_ACTIVE_SLOT(p, step);
#endif
#endif
  const int n_tiles = p.tab.n_tiles;
  const bool push = p.do_push != 0 && p.phase != 2 && comm;
  // Sticky failure: once any peer wait has timed out (this or an earlier launch) the step is a no-op on every
  // CTA -- nothing is stored into a peer that may be wedged or dead, theta stops changing, and the host raises
  // when it reads the status word.  (Uniform per CTA; the run is over, so a partial step does not matter.)
  if (p.do_push && *reinterpret_cast<volatile int*>(p.status) != EG_OK) return;

#if defined(EG_DBUF) || defined(EG_Q8) || defined(EG_GT) || defined(EG_ED)
  if (p.phase != 0 || !(p.sync && push)) return;   // the launcher rejects these; never reached
#elif defined(EG_GRAPH) || defined(EG_MATCH)
  if (p.phase != 0) return;                        // fused step only (the launcher rejects the rest)
#else
  if (p.phase == 1) {
    push_phase(p, step);
    return;
  }
#endif
  __shared__ TileInfo s_ti[EG_TI_CACHE];
  fill_tile_cache(p, s_ti);
#if !defined(EG_DBUF) && !defined(EG_GRAPH) && !defined(EG_Q8) && !defined(EG_GT) && !defined(EG_ED) && !defined(EG_MATCH)
  // spevent: receive side first -- scatter the records that arrived for this step into the replicas
  // (inbox_l / inbox_r point at them), grid barrier, then the dense mix below reads them tile by tile
  if (p.sparse != nullptr) sparse_apply_prologue(*p.sparse, p.sparse->bar);
#endif
  if (p.phase == 2 && p.sync && p.do_push) {
    // split step, second half: the neighbours' pushes of this step were issued during my backward
    __shared__ int s_pushed;
    if (tid == 0) {
      bool ok = wait_ge(p.pushed_from_l, (uint32_t)step, p.status, p.timeout_ns);
      ok = wait_ge(p.pushed_from_r, (uint32_t)step, p.status, p.timeout_ns) && ok;
      s_pushed = ok ? 1 : 0;
    }
    __syncthreads();
    if (!s_pushed) return;      // neighbour never pushed this step: do not average a stale inbox into theta
  }

  if (!(p.sync && push)) {
    // ---------------- async / split / no exchange / local step: single pass, theta read once -------
    int j = 0;
    for (int t = b; t < n_tiles; t += G, ++j) {
      const size_t base = (size_t)t * EG_TILE + (size_t)tid * EG_VEC;
      const TileInfo ti = tile_info(p, s_ti, j, t);
      const F8 th = ld_f8(p.theta + base);
      if (push && (ti.flags & 1)) push_tile(p, base, th, slot);
      mix_tile<kMom, kQG>(p, t, ti, base, th, lane, warp, step, slot, p.do_mix != 0 && comm);
    }
  } else {
    // ---------------- iter-sync: per-WARP software pipeline, no block barriers ------------------
    // Every warp owns 256 floats of each of its CTA's tiles.  It pushes its slice of tile j and
    // publishes a release-flag (tile, warp) to both neighbours, then consumes tile j-D: waits for the
    // neighbours' flags of that slice (normally long set -- the ring is symmetric) and mixes it.
    // Warps never wait for each other, so flag latency and the sys-scope fence of one warp hide
    // behind the streaming of the other 31 warps on the SM.
#if defined(EG_GRAPH)
    __shared__ int s_ok;
    if (tid == 0) {
      // WAR guard: every peer I push into must have consumed what I last pushed into its slot before I overwrite
      // it -- at step-1 on a static graph, at step-period on a one-peer graph (slot m is written every period steps);
      // with --local-steps H the last push into a slot was H (static) or period * H (one-peer) steps ago; with
      // --global-avg-period P one step ago, or two when the step before was an average (static graphs only)
      bool ok = true;
      int last = step - (p.g.period ? p.g.period : 1) * H;
      if (global_avg_step(p, step - 1)) last -= 1;
      const int prev = max(last, 0);                                       // the first round(s) wait for nothing
#pragma unroll
      for (int k = 0; k < EG_MAX_SLOTS; ++k)
        if (slot_on(p, k, slot)) ok = wait_ge(p.g.ack_from[k], (uint32_t)prev, p.status, p.timeout_ns) && ok;
      s_ok = ok;
    }
    __syncthreads();
    if (!s_ok) return;
#elif defined(EG_MATCH)
    __shared__ int s_ok;
    if (tid == 0) {
      // WAR guard: my partner has finished step k - 1, so nothing reads its inbox any more (it is written by one sender
      // per step, and only once its owner is done with the previous one)
      s_ok = wait_ge(p.m.peers[slot].done, (uint32_t)(step - 1), p.status, p.timeout_ns);
    }
    __syncthreads();
    if (!s_ok) return;
#elif !defined(EG_DBUF)
    __shared__ int s_ok;
    if (tid == 0) {
      // WAR guard: neighbours must have consumed what I pushed at step-1 (--local-steps H: at step-H, the last
      // round; --global-avg-period P: at step-2 when step-1 was an average) before I overwrite it
#if EG_LOCAL_STEPS
      const uint32_t prev = (uint32_t)max(step - H - (global_avg_step(p, step - 1) ? 1 : 0), 0);
#else
      const uint32_t prev = (uint32_t)(step - 1);
#endif
      bool ok = wait_ge(p.ack_from_l, prev, p.status, p.timeout_ns);
      ok = wait_ge(p.ack_from_r, prev, p.status, p.timeout_ns) && ok;
      s_ok = ok;
    }
    __syncthreads();
    // ack timed out (or an earlier kernel already set the sticky status): the peer may still be reading what was
    // pushed last step -- store nothing, mix nothing; the host raises on the status word
    if (!s_ok) return;
#endif
    const int D = p.group_iters;                   // pipeline depth in tiles
    const int iters = (n_tiles + G - 1) / G;
    for (int j = 0; j < iters + D; ++j) {
      const int t = b + j * G;
      if (j < iters && t < n_tiles) {
#ifdef EG_ED
        constexpr bool fired = true;               // every exact-diffusion step is a full-fire decent step
#else
        const bool fired = (tile_info(p, s_ti, j, t).flags & 1) != 0;
#endif
        if (fired) {
          const size_t base = (size_t)t * EG_TILE + (size_t)tid * EG_VEC;
#ifdef EG_DBUF
          push_tile_slot(p, base, ld_f8(p.theta + base), step);
#elif defined(EG_Q8)
          push_tile<kSign>(p, base, ld_f8(p.theta + base), slot,
                           kSign ? tile_info(p, s_ti, j, t).valid - tid * EG_VEC : EG_VEC);
#elif defined(EG_ED)
          ed_push_stage<kMom>(p, tile_info(p, s_ti, j, t), base, step);
#else
          push_tile(p, base, ld_f8(p.theta + base), slot);
#endif
        }
        __syncwarp();
        if (lane == 0) {
          if (fired) fence_sys();                  // my warp's stores are performed before the flag
#if defined(EG_GRAPH)
#pragma unroll
          for (int k = 0; k < EG_MAX_SLOTS; ++k)   // (k: out-slot; j is the tile loop's index)
            if (slot_on(p, k, slot)) st_release_sys(p.g.flag_to[k] + (size_t)t * EG_WARPS + warp, (uint32_t)step);
#elif defined(EG_MATCH)
          st_release_sys(p.m.peers[slot].flags + (size_t)t * EG_WARPS + warp, (uint32_t)step);
#elif defined(EG_Q8)
          // 2*step + fired: the receivers learn from the flag whether this block carries a delta
          const uint32_t v = 2u * (uint32_t)step + (fired ? 1u : 0u);
          st_release_sys(p.flag_to_l + (size_t)t * EG_WARPS + warp, v);
          st_release_sys(p.flag_to_r + (size_t)t * EG_WARPS + warp, v);
#else
          st_release_sys(p.flag_to_l + (size_t)t * EG_WARPS + warp, (uint32_t)step);
          st_release_sys(p.flag_to_r + (size_t)t * EG_WARPS + warp, (uint32_t)step);
#endif
        }
      }
      const int t2 = b + (j - D) * G;
      if (j >= D && t2 < n_tiles) {
#ifdef EG_Q8
        uint32_t fl = 0u, fr = 0u;
        if (lane == 0) {
          fl = wait_ge_value(p.flag_from_l + (size_t)t2 * EG_WARPS + warp, 2u * (uint32_t)step, p.status, p.timeout_ns);
          fr = wait_ge_value(p.flag_from_r + (size_t)t2 * EG_WARPS + warp, 2u * (uint32_t)step, p.status, p.timeout_ns);
        }
        __syncwarp();
        // the fired bits lane 0 observed, to the whole warp
        const int sides = __shfl_sync(0xffffffffu, (int)((fl & 1u) | ((fr & 1u) << 1)), 0);
        const size_t base = (size_t)t2 * EG_TILE + (size_t)tid * EG_VEC;
        // the CHOCO mix loads theta itself, after the replicas
        mix_tile<kMom, kQG, kSign, kChoco>(p, t2, tile_info(p, s_ti, j - D, t2), base,
                                           kChoco ? F8{} : ld_f8(p.theta + base), lane, warp, step, sides,
                                           p.do_mix != 0);
#else
        if (lane == 0) {
#ifdef EG_GRAPH
#pragma unroll
          for (int s = 0; s < EG_MAX_SLOTS; ++s)
            if (slot_on(p, s, slot))
              wait_ge(p.g.flag_from[s] + (size_t)t2 * EG_WARPS + warp, (uint32_t)step, p.status, p.timeout_ns);
#elif defined(EG_MATCH)
          wait_ge(p.m.flag_from + (size_t)t2 * EG_WARPS + warp, (uint32_t)step, p.status, p.timeout_ns);
#else
          wait_ge(p.flag_from_l + (size_t)t2 * EG_WARPS + warp, (uint32_t)step, p.status, p.timeout_ns);
          wait_ge(p.flag_from_r + (size_t)t2 * EG_WARPS + warp, (uint32_t)step, p.status, p.timeout_ns);
#endif
        }
        __syncwarp();
        const size_t base = (size_t)t2 * EG_TILE + (size_t)tid * EG_VEC;
#ifdef EG_GT
        // the tracking mix loads theta itself, after the y stage: held from here it would spill
        mix_tile<kMom, kQG>(p, t2, tile_info(p, s_ti, j - D, t2), base, F8{}, lane, warp, step, slot, p.do_mix != 0);
#elif defined(EG_ED)
        // the exact-diffusion mix loads phi itself
        mix_tile<kMom, kQG>(p, t2, tile_info(p, s_ti, j - D, t2), base, F8{}, lane, warp, step, slot, p.do_mix != 0);
#else
        mix_tile<kMom, kQG>(p, t2, tile_info(p, s_ti, j - D, t2), base, ld_f8(p.theta + base), lane, warp, step,
                            slot, p.do_mix != 0);
#endif
#endif
      }
    }
  }
  if (p.need_norm) cta_finish_tensors(p, s_ti, step + 1, p.do_mix != 0, true);
  grid_tail(p, step, slot);
}

// Quasi-global momentum needs a momentum buffer (mu > 0), iter-sync (an async mix of a stale inbox would enter m_hat),
// and no global average (the gated all-reduce overwrites theta_k before the step kernel reads it back)
static inline bool qg_rejected(const GossipParams& p) {
  return p.quasi_global != 0 && (p.mu == 0.f || p.mom == nullptr || !p.sync || p.global_avg_period != 0);
}

#if !defined(EG_DBUF) && !defined(EG_GRAPH) && !defined(EG_Q8) && !defined(EG_GT) && !defined(EG_ED) && !defined(EG_MATCH)
// (Re)compute tile partials (+ bf16 shadow) from theta (drift trigger: from theta - sent); optionally evaluate the trigger for the
// first step.  Used once at start-up and after theta is modified outside the step kernel
// (checkpoint restore).
__global__ void __launch_bounds__(EG_THREADS, 4) gossip_init_kernel(const GossipParams p, int run_fsm) {
  const int b = blockIdx.x, G = gridDim.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int next_step = *p.fsm.pass_num + 1;
  for (int t = b; t < p.tab.n_tiles; t += G) {
    const size_t base = (size_t)t * EG_TILE + (size_t)tid * EG_VEC;
    const F8 th = ld_f8(p.theta + base);
    float ss = 0.f;
    if (p.sent != nullptr) {   // drift trigger: sum (theta - sent)^2
      const F8 sv = ld_f8(p.sent + base);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float d = __fsub_rn(th.v[e], sv.v[e]);
        ss = __fmaf_rn(d, d, ss);
      }
    } else {
#pragma unroll
      for (int e = 0; e < 8; ++e) ss = __fmaf_rn(th.v[e], th.v[e], ss);
    }
    if (p.shadow != nullptr) st_bf16x8(p.shadow + base, th);
    ss = warp_sum(ss);
    if (lane == 0) {
      p.tile_ss[(size_t)t * EG_WARPS + warp] = ss;
      if (p.tile_ss_l != nullptr) {
        p.tile_ss_l[(size_t)t * EG_WARPS + warp] = 0.f;
        p.tile_ss_r[(size_t)t * EG_WARPS + warp] = 0.f;
      }
    }
  }
  if (run_fsm) cta_finish_tensors(p, nullptr, next_step, false, /*recv_ok=*/false);
}

// Trigger FSM alone, norms supplied by the caller (unit test against parallel/trigger.py).
__global__ void __launch_bounds__(EG_THREADS) fsm_decide_kernel(const FsmDev f, const TableDev t,
                                                               const float* ext_norm) {
  const int next_step = *f.pass_num + 1;
  for (int i = threadIdx.x; i < t.n_tensors; i += EG_THREADS)
    fsm_update_tensor(f, t, i, ext_norm[i], 0.f, 0.f, false, next_step, false, 2ull);
  __syncthreads();
  if (threadIdx.x == 0) *f.pass_num += 1;
}

// -------------------------------------------------------------------------------------------
int gossip_max_grid(int device) {
  int sms = 0, per_sm = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
  int per_sm2 = 0;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gossip_step_kernel<true, false>, EG_THREADS, 0);
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm2, gossip_step_kernel<false, false>, EG_THREADS, 0);
  if (per_sm2 < per_sm) per_sm = per_sm2;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm2, gossip_step_kernel<true, true>, EG_THREADS, 0);
  if (per_sm2 < per_sm) per_sm = per_sm2;
  if (per_sm < 1) per_sm = 1;
  return sms * per_sm;
}

cudaError_t launch_gossip_step(const GossipParams& p, int grid, cudaStream_t s) {
  // --local-steps: the fused dense step only (no split phases, no sparse records, no trigger, no drift copy)
  if (p.local_steps > 1 && (p.phase != 0 || p.sparse != nullptr || p.fsm.enabled || p.sent != nullptr))
    return cudaErrorInvalidValue;
  // --global-avg-period: P >= 2 (P = 1 would average at every step), on the fused dense decent step with H = 1
  if (p.global_avg_period < 0 || p.global_avg_period == 1) return cudaErrorInvalidValue;
  if (p.global_avg_period > 1 && (p.phase != 0 || p.sparse != nullptr || p.fsm.enabled || p.sent != nullptr ||
                                  p.local_steps > 1))
    return cudaErrorInvalidValue;
  if (qg_rejected(p)) return cudaErrorInvalidValue;
  eg_count_launch(EG_FAM_GOSSIP, 1);
  if (p.mu != 0.f && p.mom != nullptr)
    if (p.quasi_global)
      gossip_step_kernel<true, true><<<grid, EG_THREADS, 0, s>>>(p);
    else
      gossip_step_kernel<true, false><<<grid, EG_THREADS, 0, s>>>(p);
  else
    gossip_step_kernel<false, false><<<grid, EG_THREADS, 0, s>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_gossip_init(const GossipParams& p, int grid, int run_fsm, cudaStream_t s) {
  eg_count_launch(EG_FAM_GOSSIP, 1);
  gossip_init_kernel<<<grid, EG_THREADS, 0, s>>>(p, run_fsm);
  return cudaGetLastError();
}

cudaError_t launch_fsm_decide(const FsmDev& f, const TableDev& t, const float* ext_norm, cudaStream_t s) {
  eg_count_launch(EG_FAM_GOSSIP, 1);
  fsm_decide_kernel<<<1, EG_THREADS, 0, s>>>(f, t, ext_norm);
  return cudaGetLastError();
}

#elif defined(EG_GRAPH)   // only the step kernel + its launcher exist in this translation unit
int gossip_graph_max_grid(int device) {
  int sms = 0, a = 0, b = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&a, gossip_step_kernel_graph<true, false>, EG_THREADS, 0);
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, gossip_step_kernel_graph<false, false>, EG_THREADS, 0);
  if (b < a) a = b;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, gossip_step_kernel_graph<true, true>, EG_THREADS, 0);
  if (b < a) a = b;
  if (a < 1) a = 1;
  return sms * a;
}

// Fused decent/event step on a circulant graph: iter-sync (flags + acks per slot) or async (single pass, no flags).
// period > 0: the one-peer exponential graph, one active slot per step.
cudaError_t launch_gossip_step_graph(const GossipParams& p, const GraphSlots& g, int grid, cudaStream_t s) {
  const bool slots_ok = g.period == 0 ? (g.n_slots >= 2 && g.n_slots <= EG_MAX_SLOTS && !(g.n_slots & 1))
                                      : (g.period >= 1 && g.period <= EG_MAX_SLOTS && g.n_slots == g.period);
  if (p.phase != 0 || p.sparse != nullptr || !p.do_push || !p.do_mix || !slots_ok) return cudaErrorInvalidValue;
  if (p.local_steps > 1 && (p.fsm.enabled || p.sent != nullptr)) return cudaErrorInvalidValue;   // decent only
  // --global-avg-period: P >= 2, decent on a static graph with H = 1 (the one-peer graph's per-slot WAR bound k - tau
  // has no rule for skipped steps)
  if (p.global_avg_period < 0 || p.global_avg_period == 1) return cudaErrorInvalidValue;
  if (p.global_avg_period > 1 && (p.fsm.enabled || p.sent != nullptr || p.local_steps > 1 || g.period > 0))
    return cudaErrorInvalidValue;
  if (qg_rejected(p)) return cudaErrorInvalidValue;
  GraphStepParams q;
  static_cast<GossipParams&>(q) = p;
  q.g = g;
  eg_count_launch(EG_FAM_GOSSIP, 1);
  if (p.mu != 0.f && p.mom != nullptr)
    if (p.quasi_global)
      gossip_step_kernel_graph<true, true><<<grid, EG_THREADS, 0, s>>>(q);
    else
      gossip_step_kernel_graph<true, false><<<grid, EG_THREADS, 0, s>>>(q);
  else
    gossip_step_kernel_graph<false, false><<<grid, EG_THREADS, 0, s>>>(q);
  return cudaGetLastError();
}

#elif defined(EG_Q8)   // only the step kernel + its launcher exist in this translation unit
template <bool kMom, bool kSign, bool kChoco>
static void q8_occupancy(int& a) {
  int b = 0;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, gossip_step_kernel_q8<kMom, kSign, kChoco>, EG_THREADS, 0);
  if (b < a) a = b;
}

int gossip_q8_max_grid(int device) {   // the minimum over all eight instances
  int sms = 0, a = 1 << 30;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
  q8_occupancy<true, false, false>(a);
  q8_occupancy<false, false, false>(a);
  q8_occupancy<true, true, false>(a);
  q8_occupancy<false, true, false>(a);
  q8_occupancy<true, false, true>(a);
  q8_occupancy<false, false, true>(a);
  q8_occupancy<true, true, true>(a);
  q8_occupancy<false, true, true>(a);
  if (a < 1) a = 1;
  return sms * a;
}

template <bool kSign, bool kChoco>
static void q8_launch(const Q8StepParams& k, bool mom, int grid, cudaStream_t s) {
  if (mom)
    gossip_step_kernel_q8<true, kSign, kChoco><<<grid, EG_THREADS, 0, s>>>(k);
  else
    gossip_step_kernel_q8<false, kSign, kChoco><<<grid, EG_THREADS, 0, s>>>(k);
}

// Compressed ring step (decent/event): iter-sync fused step only.  codec 0 int8 / 1 sign; gamma 0 (the EF mix) or in
// (0, 1] (CHOCO)
cudaError_t launch_gossip_step_q8(const GossipParams& p, const Q8Slots& q, int grid, cudaStream_t s) {
  const bool ptrs = q.q_from_l && q.q_from_r && q.s_from_l && q.s_from_r && q.q_to_l && q.q_to_r && q.s_to_l &&
                    q.s_to_r && q.prev && q.rep_l && q.rep_r && p.flag_from_l && p.flag_from_r && p.flag_to_l &&
                    p.flag_to_r && p.ack_from_l && p.ack_from_r && p.ack_to_l && p.ack_to_r;
  if (p.phase != 0 || !p.sync || p.sparse != nullptr || !p.do_push || !p.do_mix || !ptrs || p.local_steps > 1 ||
      p.global_avg_period != 0 || p.quasi_global != 0)
    return cudaErrorInvalidValue;
  if (q.codec != 0 && q.codec != 1) return cudaErrorInvalidValue;
  if (!(q.gamma == 0.f || (q.gamma > 0.f && q.gamma <= 1.f))) return cudaErrorInvalidValue;   // NaN fails both
  Q8StepParams k;
  static_cast<GossipCore&>(k) = p;   // no global_avg_period, no quasi_global (refused above)
  k.q = q;
  eg_count_launch(EG_FAM_GOSSIP, 1);
  const bool mom = p.mu != 0.f && p.mom != nullptr, sign = q.codec == 1, choco = q.gamma > 0.f;
  if (sign)
    choco ? q8_launch<true, true>(k, mom, grid, s) : q8_launch<true, false>(k, mom, grid, s);
  else
    choco ? q8_launch<false, true>(k, mom, grid, s) : q8_launch<false, false>(k, mom, grid, s);
  return cudaGetLastError();
}

#elif defined(EG_GT)   // only the step kernel + its launcher exist in this translation unit
int gossip_gt_max_grid(int device) {
  int sms = 0, a = 0, b = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&a, gossip_step_kernel_gt<true>, EG_THREADS, 0);
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, gossip_step_kernel_gt<false>, EG_THREADS, 0);
  if (b < a) a = b;
  if (a < 1) a = 1;
  return sms * a;
}

// Gradient-tracking ring step (decent): iter-sync fused step only, every tensor pushed every step.
cudaError_t launch_gossip_step_gt(const GossipParams& p, const TrackSlots& y, int grid, cudaStream_t s) {
  const bool ptrs = y.y && y.g_prev && y.y_in_l && y.y_in_r && y.y_to_l &&
                    (y.y_to_r == nullptr) == (p.push_r == nullptr) && p.inbox_l && p.inbox_r && p.push_l &&
                    p.flag_from_l && p.flag_from_r && p.flag_to_l && p.flag_to_r && p.ack_from_l && p.ack_from_r &&
                    p.ack_to_l && p.ack_to_r;
  if (p.phase != 0 || !p.sync || p.sparse != nullptr || p.sent != nullptr || p.fsm.enabled || !p.do_push || !p.do_mix ||
      !p.send_ack || !ptrs || p.local_steps > 1 || p.global_avg_period != 0 || p.quasi_global != 0)
    return cudaErrorInvalidValue;
  GtStepParams k;
  static_cast<GossipCore&>(k) = p;   // no global_avg_period, no quasi_global (refused above)
  k.gt = y;
  eg_count_launch(EG_FAM_GOSSIP, 1);
  if (p.mu != 0.f && p.mom != nullptr)
    gossip_step_kernel_gt<true><<<grid, EG_THREADS, 0, s>>>(k);
  else
    gossip_step_kernel_gt<false><<<grid, EG_THREADS, 0, s>>>(k);
  return cudaGetLastError();
}

#elif defined(EG_ED)   // only the step kernel + its launcher exist in this translation unit
int gossip_ed_max_grid(int device) {
  int sms = 0, a = 0, b = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&a, gossip_step_kernel_ed<true>, EG_THREADS, 0);
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, gossip_step_kernel_ed<false>, EG_THREADS, 0);
  if (b < a) a = b;
  if (a < 1) a = 1;
  return sms * a;
}

// Exact-diffusion ring step (decent): iter-sync fused step only, every tensor pushed every step.
cudaError_t launch_gossip_step_ed(const GossipParams& p, const EdSlots& e, int grid, cudaStream_t s) {
  const bool ptrs = e.psi && p.inbox_l && p.inbox_r && p.push_l && p.flag_from_l && p.flag_from_r && p.flag_to_l &&
                    p.flag_to_r && p.ack_from_l && p.ack_from_r && p.ack_to_l && p.ack_to_r;
  if (p.phase != 0 || !p.sync || p.sparse != nullptr || p.sent != nullptr || p.fsm.enabled || !p.do_push || !p.do_mix ||
      !p.send_ack || !ptrs || p.local_steps > 1 || p.global_avg_period != 0 || p.quasi_global != 0)
    return cudaErrorInvalidValue;
  EdStepParams k;
  static_cast<GossipCore&>(k) = p;   // no global_avg_period, no quasi_global (refused above)
  k.ed = e;
  eg_count_launch(EG_FAM_GOSSIP, 1);
  if (p.mu != 0.f && p.mom != nullptr)
    gossip_step_kernel_ed<true><<<grid, EG_THREADS, 0, s>>>(k);
  else
    gossip_step_kernel_ed<false><<<grid, EG_THREADS, 0, s>>>(k);
  return cudaGetLastError();
}

#elif defined(EG_MATCH)   // only the step kernel + its launcher exist in this translation unit
int gossip_match_max_grid(int device) {
  int sms = 0, a = 0, b = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&a, gossip_step_kernel_match<true>, EG_THREADS, 0);
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, gossip_step_kernel_match<false>, EG_THREADS, 0);
  if (b < a) a = b;
  if (a < 1) a = 1;
  return sms * a;
}

// Random-match step (decent): iter-sync fused step only, every tensor pushed to the step's partner.
cudaError_t launch_gossip_step_match(const GossipParams& p, const MatchSlots& m, int grid, cudaStream_t s) {
  const bool ok = m.world >= 2 && m.world <= EG_MATCH_MAX_WORLD && m.rank >= 0 && m.rank < m.world && m.seed >= 0 &&
                  m.peers && m.inbox && m.flag_from && m.done;
  if (p.phase != 0 || !p.sync || p.sparse != nullptr || p.sent != nullptr || p.fsm.enabled || !p.do_push ||
      !p.do_mix || !p.send_ack || !ok || p.local_steps > 1 || p.global_avg_period != 0 || p.quasi_global != 0)
    return cudaErrorInvalidValue;
  MatchStepParams k;
  static_cast<GossipParams&>(k) = p;
  k.m = m;
  eg_count_launch(EG_FAM_GOSSIP, 1);
  if (p.mu != 0.f && p.mom != nullptr)
    gossip_step_kernel_match<true><<<grid, EG_THREADS, 0, s>>>(k);
  else
    gossip_step_kernel_match<false><<<grid, EG_THREADS, 0, s>>>(k);
  return cudaGetLastError();
}

#else   // EG_DBUF: only the step kernel + its launcher exist in this translation unit
int gossip_dbuf_max_grid(int device) {
  int sms = 0, a = 0, b = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&a, gossip_step_kernel_dbuf<true, false>, EG_THREADS, 0);
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, gossip_step_kernel_dbuf<false, false>, EG_THREADS, 0);
  if (b < a) a = b;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, gossip_step_kernel_dbuf<true, true>, EG_THREADS, 0);
  if (b < a) a = b;
  if (a < 1) a = 1;
  return sms * a;
}

// Dense iter-sync exchange only (decent): every tensor fires every step, inboxes hold 2 slots.
cudaError_t launch_gossip_step_dbuf(const GossipParams& p, int grid, cudaStream_t s) {
  if (p.phase != 0 || !p.sync || !p.do_push || !p.do_mix || p.fsm.enabled || p.sent != nullptr || p.local_steps > 1 ||
      p.global_avg_period != 0 || qg_rejected(p))
    return cudaErrorInvalidValue;
  eg_count_launch(EG_FAM_GOSSIP, 1);
  if (p.mu != 0.f && p.mom != nullptr)
    if (p.quasi_global)
      gossip_step_kernel_dbuf<true, true><<<grid, EG_THREADS, 0, s>>>(p);
    else
      gossip_step_kernel_dbuf<true, false><<<grid, EG_THREADS, 0, s>>>(p);
  else
    gossip_step_kernel_dbuf<false, false><<<grid, EG_THREADS, 0, s>>>(p);
  return cudaGetLastError();
}
#endif

}  // namespace egb
