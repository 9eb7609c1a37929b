// eventgrad_b200 -- host-visible launch API of the sm_90a kernels.
// Pure CUDA (no torch headers) so the .cu files compile in seconds; bindings.cpp adapts tensors.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>

#include <utility>
#include <vector>

#define EG_TILE 2048     // fp32 elements per tile == parallel/arena.py:TILE
#define EG_THREADS 256
#define EG_MAX_SLOTS 8   // inbox slots of a circulant gossip graph: 2 per offset, <= 4 offsets (parallel/topology.py)
#define EG_MATCH_MAX_WORLD 1024   // random-match: ranks of the matching (its shuffle is kept in shared memory)

namespace egb {

// ------------------------------------------------------------------ launch accounting (host)
// Every launcher of this extension counts the kernels it enqueues (per family), so "how many of OUR kernels ran
// in this region" is counted, not derived from a formula (bench.py `gpu_launches`; during CUDA-graph capture the
// Trainer records the per-step delta and multiplies by the replays).
enum { EG_FAM_GOSSIP = 0, EG_FAM_ALLREDUCE, EG_FAM_SPARSE, EG_FAM_BN, EG_FAM_LINEAR, EG_FAM_DATA, EG_FAM_CONV, EG_FAM_N };
void eg_count_launch(int family, int n);

// ------------------------------------------------------------------ tensor table (device)
struct TableDev {
  const int* tile_tensor;   // [n_tiles]  tile -> parameter tensor
  const int* t_tile_start;  // [n_tensors]
  const int* t_tile_count;  // [n_tensors]
  const int* t_numel;       // [n_tensors]
  const int* t_msg_bytes;   // [n_tensors] bytes one neighbour receives when tensor i fires
  int n_tiles;
  int n_tensors;
};

// ------------------------------------------------------------------ event-trigger FSM (device)
// Mirrors /root/reference/dcifar10/event/event.cpp:300-365 -- see parallel/trigger.py (oracle).
struct FsmDev {
  float* thres;        // [sz]
  float* last_norm;    // [sz]
  float* last_iter;    // [sz]
  float* slopes;       // [sz * history]
  int* fire;           // [sz] decision for the step that is about to run
  float* cur_norm;     // [sz] sender norm used for that decision
  unsigned long long* counters;  // [0] events (+2 per fire)  [1] payload bytes pushed  [2] fired tensors
  int* pass_num;       // completed steps (device-resident so CUDA graphs can replay the step)
  float* log_ring;     // optional [log_cap][sz][5] = norm, thres, fired, left_norm, right_norm
  int log_cap;
  float horizon;
  float constant;
  int thres_type;      // 1 adaptive, 0 constant
  int history;         // sent_history (<= 8)
  int initial_comm_passes;
  int enabled;         // 0: decent / cent (no trigger: fire[] stays all-ones)
  int metric;          // trigger input: 0 norm difference | ||theta|| - ||theta at last send|| | (reference),
                       // 1 drift ||theta - sent|| from what the receivers hold (GossipParams.sent); cur_norm holds it
};

struct SparseParams;
// ------------------------------------------------------------------ fused gossip step
// One launch = push theta_k to both ring neighbours (only tensors whose trigger fired) ->
// [iter-sync: flag handshake] -> (theta+L+R)/3 -> SGD(+momentum) -> write theta_{k+1} (+bf16
// shadow, zero grad) accumulating per-warp sum-of-squares -> last CTA evaluates the trigger FSM
// for step k+1 from those partials.  Replaces, per step, 86x{norm.item(), 2 MPI_Put, 2 memcpy,
// add_, add_, div_} + optimizer.step() of the reference.
// GossipCore is the block every step kernel reads; GossipParams appends the fields that only the ring and graph kernels
// read.  The int8, tracking and exact-diffusion kernels take GossipCore followed by their own slots (their launchers
// slice it out of GossipParams), so those slots keep the offsets they had when GossipCore was all of GossipParams.
struct GossipCore {
  float* theta;
  float* grad;
  float* mom;               // may be null when mu == 0
  const float* inbox_l;     // local: what my LEFT neighbour last pushed (or its sparse replica)
  const float* inbox_r;
  float* push_l;            // peer-mapped: LEFT neighbour's inbox_r
  float* push_r;            // peer-mapped: RIGHT neighbour's inbox_l
  __nv_bfloat16* shadow;    // optional bf16 copy of theta_{k+1} for the next forward
  const void* const* t_grad_ptr;  // optional [sz]: read each tensor's gradient in place (table mode)
  const int* t_grad_bf16;         // [sz] 1: that gradient is bf16, 0: fp32
  float* tile_ss;           // [n_tiles * 8] per-warp sum theta_{k+1}^2
  float* tile_ss_l;         // optional (logging): sum inbox_l^2
  float* tile_ss_r;
  // iter-sync handshake (all monotonic step counters)
  uint32_t* flag_from_l;    // local, written by left neighbour   [n_tiles * 8] (tile, warp)
  uint32_t* flag_from_r;
  uint32_t* flag_to_l;      // peer-mapped: left neighbour's flag_from_r
  uint32_t* flag_to_r;      // peer-mapped: right neighbour's flag_from_l
  uint32_t* ack_from_l;     // local: left neighbour finished reading what I pushed at step k
  uint32_t* ack_from_r;
  uint32_t* ack_to_l;       // peer-mapped
  uint32_t* ack_to_r;
  uint32_t* pushed_from_l;  // split step: left neighbour has finished ALL its pushes of step k
  uint32_t* pushed_from_r;
  uint32_t* pushed_to_l;    // peer-mapped
  uint32_t* pushed_to_r;
  unsigned int* ticket;     // [0] last-CTA election (step) [1] push phase
  unsigned int* tensor_done; // [sz] per-tensor count of per-warp partials written this launch
  int* status;              // sticky error word
  unsigned long long timeout_ns;
  TableDev tab;
  FsmDev fsm;
  float lr;
  float mu;
  int do_mix;               // 0: plain SGD (serial run)
  int do_push;              // 0: sparse mode (records are pushed by the top-k kernels) / serial
  int sync;                 // 1: iter-sync handshake, 0: async (reference RMA semantics)
  int send_ack;             // sync: write acks in the tail (0 when another kernel acks)
  int zero_grad;
  int group_iters;          // iter-sync software-pipeline depth in tiles (push j, mix j-D)
  const struct SparseParams* sparse;   // spevent: device copy of the sparse parameters -> the kernel's prologue scatters
                            // the arrived (value, index) records into inbox_l / inbox_r (the replicas) first
  int need_norm;            // 0: skip norm-on-write + trigger entirely (decent/cent without logs)
  int phase;                // 0 fused step | 1 push only (side stream, overlaps backward) | 2 wait+mix+SGD
  // optimizer options (torch.optim.SGD semantics, applied after the mix; see sgd_elem in common.cuh)
  float wd;                 // weight decay, every arena tensor (0: off)
  int nesterov;             // 1: Nesterov momentum (needs mu > 0)
  const float* lr_table;    // optional [lr_len]: lr of step s is lr_table[min(s-1, lr_len-1)]; null: the scalar lr
  int lr_len;
  // periodic gossip (--local-steps H, decent on the ring and on graphs): step k gossips iff H divides k, every other
  // step is the serial SGD step (no push, no flag, no ack, no mix).  0 or 1: every step gossips.  It sits in the padding
  // in front of `sent`, so the size of this block and the offset of every other field are unchanged
  int local_steps;
  // drift trigger (fsm.metric = 1): what the receivers hold of theta.  event: every pushed tile also stores theta_k
  // here, and the norm-on-write partials are sum (theta_{k+1} - sent)^2; spevent: the sparse `prev` (written by the
  // compaction, never by the step kernel).  null: the norm rule, no extra loads or stores
  float* sent;
};

struct GossipParams : GossipCore {
  // periodic global averaging (--global-avg-period P >= 2, decent on the ring and on static graphs): at step k with P
  // dividing k the gated all-reduce launched just before the step kernel has already replaced theta by the rank mean,
  // and the step kernel takes the plain SGD step (no push, no flag, no ack, no mix).  0: off.  The WAR guard of the
  // next gossip step waits for the ack of k - 1 (PROTOCOL.md 1.11)
  int global_avg_period;
  // quasi-global momentum (--quasi-global-momentum, decent/event/spevent on the ring, the double-buffered ring and
  // circulant / one-peer graphs; needs mu > 0 and iter-sync): `mom` holds m_hat, built from the step's own parameter
  // displacement theta_k - theta_{k+1} instead of the gradient (qg_sgd_elem in common.cuh).  0: the plain sgd_elem.
  // It fills the tail padding after global_avg_period, so the size of this block is unchanged
  int quasi_global;
};
static_assert(sizeof(GossipParams) == sizeof(GossipCore) + 8, "GossipParams: global_avg_period and quasi_global fill "
                                                              "the 8 bytes after GossipCore");

// Circulant gossip graph beyond the ring (csrc/gossip_graph.cu): the 2|O| inbox slots that replace the ring's
// left/right pointers.  A separate block, passed to the graph kernel next to GossipParams, so the ring kernels'
// parameters are untouched.  Slot s of this rank receives from peer Graph.slots()[s]; out-slot j pushes into slot j of
// peer Graph.out_slots()[j] (parallel/topology.py).  mix: theta <- (((theta + in_0) + in_1) + ...) / (n_slots + 1)
// period > 0: the time-varying one-peer exponential graph (OnePeerExp): slot m receives from r - 2^m, and at step k only
// slot m = (k-1) % period takes part (push, flag, ack), with the mix theta <- (theta + in_m) / 2.  The kernel derives m
// from the device step counter, so one captured launch serves every step of the cycle.
struct GraphSlots {
  int n_slots;                          // static: 2|O|, even, 2..EG_MAX_SLOTS; one-peer: period, 1..EG_MAX_SLOTS
  int period;                           // 0: static circulant graph; > 0: one-peer graph with n_slots == period
  const float* inbox[EG_MAX_SLOTS];     // local: what the sender of slot s last pushed
  float* push[EG_MAX_SLOTS];            // peer-mapped: slot j's inbox of my j-th out peer
  uint32_t* flag_from[EG_MAX_SLOTS];    // local [n_tiles * 8] (tile, warp), written by the sender of slot s
  uint32_t* flag_to[EG_MAX_SLOTS];      // peer-mapped: flag_from[j] of my j-th out peer
  uint32_t* ack_from[EG_MAX_SLOTS];     // local: my j-th out peer finished reading what I pushed at step k
  uint32_t* ack_to[EG_MAX_SLOTS];       // peer-mapped: ack_from[s] of the sender of slot s
};

// Random pairwise matchings (csrc/gossip_match.cu, --topology random-match, decent): a separate block passed to the match
// kernel next to GossipParams, whose ring pointers it leaves unused.  At step k = *pass_num + 1 thread 0 of every CTA
// derives the partner p from (seed, world, k) (parallel/topology.py match_pairs: splitmix64 from (seed << 32) ^ k,
// Fisher-Yates, pairs (pi[0], pi[1]), ...).  A matched rank waits for peers[p].done >= k - 1 (p has finished step k - 1,
// so its single inbox is free), pushes theta_k into peers[p].inbox with one (tile, warp) flag = k in peers[p].flags,
// waits for its own flag_from = k and mixes theta <- (theta + inbox) / 2; an idle rank (odd world) takes the plain SGD
// step.  The last CTA stores *done = k on every rank (PROTOCOL.md 1.17).
struct MatchPeer {
  float* inbox;             // peer-mapped: that rank's single inbox [n_padded]
  uint32_t* flags;          // peer-mapped: that rank's (tile, warp) flag block [n_tiles * 8]
  const uint32_t* done;     // peer-mapped: the last step that rank has finished
};
struct MatchSlots {
  int world;                // 2 .. EG_MATCH_MAX_WORLD
  int rank;
  int seed;                 // [0, 2^31)
  const MatchPeer* peers;   // device array [world], built once by the backend
  const float* inbox;       // local: what this step's partner pushed
  uint32_t* flag_from;      // local [n_tiles * 8]: written by this step's partner
  uint32_t* done;           // local: the last step this rank has finished (read by every partner)
};

// int8 error-feedback compression of the ring's pushes (csrc/gossip_q8.cu, --compress int8): a separate block passed
// to the q8 kernel next to GossipParams, which keeps its ring flag / ack pointers.  Per fired tile each warp sends the
// int8 code of theta - prev for its 256 elements (one 8-byte store per lane and neighbour) and one fp32 scale, adds the
// dequantized delta to `prev`, and its receivers add the same delta to their replica of it; the mix reads the
// replicas: theta <- ((theta + rep_l) + rep_r) / 3.  The codec (parallel/trigger.py q8_encode) is
// s = max|d| / 127, q = s == 0 ? 0 : clamp(rint(d / s), -127, 127), deq = q * s, all IEEE round-to-nearest.
// codec = 1 (--compress sign) replaces it by a 1-bit scaled sign on the same (tile, warp) block of 256 elements
// (parallel/trigger.py sign_encode): each lane sums its 8 values of |d| left to right, the warp adds a + shfl_xor(a, o)
// for o = 16, 8, 4, 2, 1, s = a / 256 (true division); bit e of the lane's byte is d_e < 0 and deq_e = bit ? -s : s.
// Lane j of block b writes byte 32 b + j (= base >> 3) of the code inbox and the scale goes where int8's does, so the
// sign path uses 1/8 of the code section.
// gamma > 0 (--choco-gamma, CHOCO-SGD) replaces the mix by the consensus step on the public copies, after this step's
// push has updated prev and the receive side the replicas (parallel/trigger.py choco_mix_):
//   t = ((prev + rep_l) + rep_r) / 3,  theta <- theta + gamma * (t - prev)
// which keeps the sum of theta over the ranks whatever the codec.  gamma = 0: the mix above.  The push, the flags,
// prev and the replica updates are the same for both mixes.
struct Q8Slots {
  const int8_t* q_from_l;   // local [n_tiles * EG_TILE] codes last pushed by my LEFT neighbour
  const int8_t* q_from_r;
  const float* s_from_l;    // local [n_tiles * 8] one scale per (tile, warp) block
  const float* s_from_r;
  int8_t* q_to_l;           // peer-mapped: LEFT neighbour's q_from_r
  int8_t* q_to_r;           // peer-mapped: RIGHT neighbour's q_from_l
  float* s_to_l;
  float* s_to_r;
  float* prev;              // what my neighbours hold of my theta (dequantized public copy)
  float* rep_l;             // my copy of my LEFT neighbour's prev
  float* rep_r;
  int codec;                // 0: int8, 1: scaled sign (appended last, so no existing offset moves)
  float gamma;              // 0: the mix ((theta + rep_l) + rep_r) / 3; (0, 1]: the CHOCO consensus step
};

// Gradient tracking for decent on the ring (csrc/gossip_gt.cu, --gradient-tracking): a separate block passed to the
// tracking kernel next to GossipParams, which keeps its ring inbox / push / flag / ack pointers for theta.  Each rank
// also gossips y, which tracks the average gradient, and steps along it:
//   push  theta_k and y_{k-1} to both neighbours (same thread, before the same (tile, warp) flag)
//   y_k = ((y_{k-1} + yL) + yR) / 3 + (g_k - g_{k-1}),  g_prev <- g_k,  theta' = ((theta_k + L) + R) / 3,
//   theta_{k+1} = sgd_elem(theta', y_k, ...)
// 2-rank ring: y_to_r is null and y_in_l == y_in_r, exactly as push_r / inbox_l of the single-copy wire dedup.
struct TrackSlots {
  float* y;                 // local: y_{k-1} before the step, y_k after it
  float* g_prev;            // local: the gradient of the previous step (fp32, also when the gradient is bf16)
  const float* y_in_l;      // local: y last pushed by my LEFT neighbour
  const float* y_in_r;
  float* y_to_l;            // peer-mapped: LEFT neighbour's y_in_r
  float* y_to_r;            // peer-mapped: RIGHT neighbour's y_in_l (null on the 2-rank ring)
};

// Exact diffusion for decent on the ring (csrc/gossip_ed.cu, --exact-diffusion): D^2 on W_bar = (I + W) / 2.  A
// separate block passed to the ED kernel next to GossipParams, which keeps its ring inbox / push / flag / ack pointers;
// the pushed message is phi instead of theta:
//   push  p = sgd_elem(theta_k, g_k, ...),  phi = p + (theta_k - psi),  psi <- p,  phi to both neighbours and to theta
//   theta_{k+1} = (phi + ((phi + L) + R) / 3) / 2
struct EdSlots {
  float* psi;               // local: the previous optimizer output p (theta_0 before the first step)
};

int gossip_max_grid(int device);  // co-resident CTAs (persistent grid upper bound)
cudaError_t launch_gossip_step(const GossipParams& p, int grid, cudaStream_t s);
// experimental double-buffered dense variant (csrc/gossip_dbuf.cu): inbox_l/inbox_r/push_l/push_r address
// TWO consecutive slots of n_tiles*EG_TILE floats; requires phase 0, sync, do_push, do_mix, fsm disabled
// experimental copy-engine push of the split step (csrc/ce_push.cu): ack wait -> 2 x cudaMemcpyAsync -> flags
cudaError_t launch_ce_push(const GossipParams& p, cudaStream_t s);
int gossip_dbuf_max_grid(int device);
cudaError_t launch_gossip_step_dbuf(const GossipParams& p, int grid, cudaStream_t s);
// circulant-graph step (csrc/gossip_graph.cu): the fused single-kernel step over the slots of `g`; requires phase 0,
// no sparse block, do_push and do_mix, and an even n_slots in [2, EG_MAX_SLOTS] (static) or n_slots == period in
// [1, EG_MAX_SLOTS] (one-peer)
int gossip_graph_max_grid(int device);
cudaError_t launch_gossip_step_graph(const GossipParams& p, const GraphSlots& g, int grid, cudaStream_t s);
// random-match step (csrc/gossip_match.cu): the fused single-kernel decent step over the single inbox of `m`; requires
// phase 0, sync, do_push, do_mix and send_ack, no sparse block, no `sent`, the trigger off, local_steps <= 1, no global
// averaging or quasi-global momentum, and every pointer of `m`
int gossip_match_max_grid(int device);
cudaError_t launch_gossip_step_match(const GossipParams& p, const MatchSlots& m, int grid, cudaStream_t s);
// int8-compressed ring step (csrc/gossip_q8.cu): the fused single-kernel step with the pushes, replicas and flags of
// `q`; requires phase 0, sync, do_push and do_mix, no sparse block, every pointer of `q` set, codec 0 or 1 and gamma 0
// or in (0, 1].  The iter-sync flag of (tile, warp) carries 2*step + fired (PROTOCOL.md 1.7, 1.15)
int gossip_q8_max_grid(int device);
cudaError_t launch_gossip_step_q8(const GossipParams& p, const Q8Slots& q, int grid, cudaStream_t s);
// gradient-tracking ring step (csrc/gossip_gt.cu): the fused single-kernel decent step that also gossips y and steps
// along it; requires phase 0, sync, do_push and do_mix, no sparse block, no `sent`, the ring's inbox / push / flag /
// ack pointers and every pointer of `y` (y_to_r null exactly when push_r is null)
int gossip_gt_max_grid(int device);
cudaError_t launch_gossip_step_gt(const GossipParams& p, const TrackSlots& y, int grid, cudaStream_t s);
// exact-diffusion ring step (csrc/gossip_ed.cu): the fused single-kernel decent step that runs the optimizer in the push
// stage and gossips phi; requires phase 0, sync, do_push, do_mix and send_ack, no sparse block, no `sent`, the trigger
// off, local_steps <= 1, the ring's inbox / push / flag / ack pointers and `psi`
int gossip_ed_max_grid(int device);
cudaError_t launch_gossip_step_ed(const GossipParams& p, const EdSlots& e, int grid, cudaStream_t s);
// Mix-only gossip rounds (csrc/gossip_rounds.cu, --gossip-rounds Q >= 2, decent on the ring or a static circulant
// graph): `rounds` = Q - 1 launches of one round each, enqueued after backward and before the step kernel.  Round q of
// step k = *pass_num + 1 pushes theta into every out-slot's round inbox, flags and acks with h = rounds * (k - 1) + q,
// and mixes theta <- (((theta + in_0) + in_1) + ...) / (n_slots + 1) in place.  Its own parameter block and window
// sections (slot s of this rank receives from Graph.slots()[s]; out-slot j pushes into slot j of Graph.out_slots()[j]),
// so no step kernel's parameters change.  2-rank ring: push[0] is null and inbox[0] == inbox[1] (one copy on the wire)
struct RoundParams {
  float* theta;
  const int* pass_num;                  // completed steps (the gossip pass counter the step kernel advances)
  unsigned int* ticket;                 // [1] last-CTA election of this kernel only
  int* status;                          // sticky error word
  unsigned long long timeout_ns;
  int n_tiles;
  int group_iters;                      // per-warp pipeline depth in tiles, as the step kernel's
  int rounds;                           // Q - 1 >= 1
  int n_slots;                          // 2 (ring) or 2|O|: even, 2..EG_MAX_SLOTS
  const float* inbox[EG_MAX_SLOTS];     // local: round inbox of slot s
  float* push[EG_MAX_SLOTS];            // peer-mapped: slot j's round inbox of my j-th out peer (null: not sent)
  uint32_t* flag_from[EG_MAX_SLOTS];    // local [n_tiles * 8] (tile, warp), written by the sender of slot s
  uint32_t* flag_to[EG_MAX_SLOTS];      // peer-mapped: flag_from[j] of my j-th out peer
  uint32_t* ack_from[EG_MAX_SLOTS];     // local: my j-th out peer finished reading my round h push
  uint32_t* ack_to[EG_MAX_SLOTS];       // peer-mapped: ack_from[s] of the sender of slot s
};
int gossip_rounds_max_grid(int device);  // co-resident CTAs (persistent grid upper bound)
// the p.rounds launches of one step, q = 1 .. rounds, on stream s
cudaError_t launch_gossip_rounds(const RoundParams& p, int grid, cudaStream_t s);
// Chebyshev-accelerated rounds (--gossip-accel chebyshev): the same RoundParams with `rounds` = Q (every round is a
// round launch; the step kernel after them runs as the serial step), plus this block.  Round q keeps x_{q-1}, the theta
// it loads, forms the round's mix w, and stores
//   x_q = (x_{q-1} + alpha_q (w - x_{q-1})) + omega_q (x_{q-1} - x_{q-2})      (q = 1: no omega term, prev not read)
// into theta, and x_{q-1} into prev for q < Q.  coef[2 (q - 1)] = alpha_q, coef[2 (q - 1) + 1] = omega_q, fp32
// (parallel/topology.py chebyshev_coefficients)
struct ChebParams {
  float* prev;                          // local [n_padded]: x_{q-1} of the previous round
  const float* coef;                    // device [Q][2]: (alpha_q, omega_q)
};
cudaError_t launch_gossip_rounds_cheb(const RoundParams& p, const ChebParams& c, int grid, cudaStream_t s);
// (re)compute tile_ss (+ shadow) from theta and evaluate the trigger for step pass_num+1.
cudaError_t launch_gossip_init(const GossipParams& p, int grid, int run_fsm, cudaStream_t s);
// Trigger FSM alone with externally supplied norms (unit tests against the oracle).
cudaError_t launch_fsm_decide(const FsmDev& f, const TableDev& t, const float* ext_norm, cudaStream_t s);

// ------------------------------------------------------------------ one-/two-shot all-reduce
// cent: grad <- sum_r grad_r / R fused with the SGD step; also final parameter averaging.
struct AllReduceParams {
  float* const* peer_bufs;  // device array [world] of peer-mapped pointers to the SAME buffer on each rank
  float* local;             // == peer_bufs[rank]
  float* theta;             // SGD mode: parameters (may alias nothing in `local`)
  float* mom;
  __nv_bfloat16* shadow;
  uint32_t* const* peer_flags;  // device array [world]: each rank's flag block (peer-mapped)
  uint32_t* flags;              // local flag block: [3][grid][world]
  unsigned int* ticket;
  int* status;
  int* step_ctr;            // device-resident launch counter for the flag protocol
  unsigned long long timeout_ns;
  int n_tiles;
  int rank;
  int world;
  float lr;
  float mu;
  int mode;                 // 0: average in place   1: average + SGD (+ zero grad)
  int two_shot;             // 0: every rank reads all peers   1: reduce-scatter + broadcast
  int zero_after;
  float* mc_local;          // NVLS variant only: multicast (NVSwitch) mapping of `local`; null otherwise
  // SGD mode: optimizer options as in GossipParams, and the rank's device pass counter (the step index into
  // lr_table), advanced once per launch in the tail.  pass_num null: not advanced (averaging mode).
  float wd;
  int nesterov;
  const float* lr_table;
  int lr_len;
  int* pass_num;
  // step gate (--global-avg-period): gate_period > 0 makes every CTA read *gate_pass + 1, the 1-based step about to
  // run, and return before its first cross-rank barrier unless gate_period divides it -- without touching step_ctr or
  // the ticket, so a skipped launch leaves no trace.  gate_pass is the rank's gossip pass counter, which iter-sync keeps
  // equal on every rank, so every rank skips the same launches.  0: every launch averages
  const int* gate_pass;
  int gate_period;
};
cudaError_t launch_allreduce(const AllReduceParams& p, int grid, cudaStream_t s);
// SlowMo (--slowmo-period tau, decent; csrc/allreduce.cu): the all-reduce block followed by the outer iterate x and
// the slow momentum u (arena-sized, local device memory, identical on every rank) and the slow momentum / learning rate.
// The sync kernel is gated like the --global-avg-period all-reduce (gate_pass, gate_period = tau): at step k with tau
// dividing k it averages theta two-shot into every rank's theta window, then every rank applies, tile by tile,
//   lr != 0:  u <- beta*u + (x - theta_bar) / lr ;  x <- fma(u, -alpha*lr, x)        lr == 0:  x <- theta_bar
// and stores theta <- x (and the bf16 shadow when set).  A separate struct, so AllReduceParams and the all-reduce
// instances keep their layout and code
struct SlowMoParams : AllReduceParams {
  float* x;
  float* u;
  float beta;
  float alpha;
};
cudaError_t launch_slowmo_sync(const SlowMoParams& p, int grid, cudaStream_t s);
// Consensus distance (--consensus-every N; csrc/allreduce.cu): the all-reduce block (two-shot, peer_bufs = every
// rank's theta, gate_pass = the gossip pass counter, gate_period = N) followed by the arena's tensor table, the
// partial buffers and the measurement ring.  After step k with N dividing k (k = *gate_pass, the step that just
// completed) every tile owner forms theta_bar with reduce_tile's rounding and, over the tile's real elements, in fp64,
//   D = sum_r (theta_r - theta_bar)^2        A = theta_bar^2
// per (tile, warp); it stores both into every rank's partial buffer, and the last CTA of every rank reduces them per
// tensor into ring row (*ring_ctr mod cap): [n_tensors][2] doubles, ring_step[row] = k.  theta is only read.  A
// separate struct, so AllReduceParams and the all-reduce instances keep their layout and code
struct ConsensusParams : AllReduceParams {
  double* const* peer_part;  // device array [world]: each rank's partial buffer [n_tiles][EG_WARPS][2] (peer-mapped)
  const double* part;        // == peer_part[rank]
  const int* tile_tensor;    // [n_tiles]
  const int* t_tile_start;   // [n_tensors]
  const int* t_tile_count;
  const int* t_numel;
  int n_tensors;
  double* ring;              // [cap][n_tensors][2] (local)
  int* ring_step;            // [cap]
  int* ring_ctr;             // measurements written so far
  int cap;
};
int consensus_max_grid(int device);  // co-resident CTAs; also loads the kernel before any step kernel spins
cudaError_t launch_consensus(const ConsensusParams& p, int grid, cudaStream_t s);
// experimental NVLink-SHARP variant (csrc/allreduce_nvls.cu): multimem.ld_reduce + multimem.st, two-shot only
cudaError_t launch_allreduce_nvls(const AllReduceParams& p, int grid, cudaStream_t s);

// ------------------------------------------------------------------ sparse (top-k) exchange
struct SparseParams {
  const float* theta;
  float* prev;              // what this rank last sent (element-wise)
  float* rep_l;             // persistent replicas of the neighbours
  float* rep_r;
  // records: per tensor [vals(k_i) | idx(k_i)] at rec_off[i] (4-byte words)
  const float* rec_from_l;  // local inbox records written by neighbours
  const float* rec_from_r;
  float* rec_to_l;          // peer-mapped: left neighbour's rec_from_r
  float* rec_to_r;          // peer-mapped: right neighbour's rec_from_l
  uint32_t* seq_from_l;     // [sz] local: step at which the record of tensor i was last rewritten
  uint32_t* seq_from_r;
  uint32_t* seq_to_l;       // peer-mapped
  uint32_t* seq_to_r;
  uint32_t* applied_l;      // [sz] local bookkeeping: last seq applied to the replica
  uint32_t* applied_r;
  uint32_t* done_from_l;    // sync: neighbour finished writing all records of step k
  uint32_t* done_from_r;
  uint32_t* done_to_l;
  uint32_t* done_to_r;
  uint32_t* ack_from_l;
  uint32_t* ack_from_r;
  uint32_t* ack_to_l;
  uint32_t* ack_to_r;
  const int* t_k;           // [sz] k_i
  const int* t_rec_off;     // [sz] record offset (words)
  // scratch
  unsigned int* hist;       // [sz][2048] (left all-zero by every launch)
  unsigned int* sel_prefix; // [sz] pass 1: top 11 bits of tau; after pass 2: tau = the k-th largest |diff| key
  unsigned int* sel_remain; // [sz] pass 1: rank inside the bucket; after pass 2: number of keys == tau to select
  uint32_t* cand;           // [n_tiles * EG_TILE] candidate keys (low 21 bits), tensor i at t_tile_start[i]*EG_TILE
  unsigned int* cand_cnt;   // [sz]
  unsigned int* done1;      // [sz] per-tensor tile-completion counters of pass 1 / pass 2
  unsigned int* done2;
  unsigned long long* desc; // [n_tiles] look-back descriptors of pass 3
  unsigned int* bar;        // [2] grid barrier of the receive prologue (arrivals, generation)
  const int* fire;
  const int* pass_num;
  unsigned int* ticket;
  int* status;
  unsigned long long timeout_ns;
  TableDev tab;
  int sync;
};
// 3 launches: histogram+pick, candidates+exact threshold, ordered compaction straight into the neighbours' inboxes.
// `grid` must be a co-resident persistent grid (pass 3 uses a decoupled look-back between CTAs).
cudaError_t launch_sparse_select_push(const SparseParams& p, int grid, cudaStream_t s);
cudaError_t launch_sparse_apply(const SparseParams& p, int grid, cudaStream_t s);

// ------------------------------------------------------------------ data path
// uint8 NCHW batch -> normalised fp32/bf16 (NCHW or NHWC) with pad+flip+crop folded in.
cudaError_t launch_decode_augment(const uint8_t* in, void* out, const int* oy, const int* ox,
                                  const int* flip, int B, int C, int H, int W, int pad, float scale,
                                  float mean, float inv_std, int out_bf16, int nhwc, cudaStream_t s);

// ------------------------------------------------------------------ fused BatchNorm(+add)(+ReLU)
// NHWC activations [M = N*H*W, C] in fp32 (reference precision) or bf16, fp32 statistics / affine parameters
// (csrc/bn_act.cu).
struct BnParams {
  const void* x;              // BN input (conv output)
  const void* res;            // optional residual added before the activation
  void* y;                    // output (forward) / saved output for the ReLU mask (backward)
  const void* dy;             // backward: grad wrt y
  void* dx;                   // backward: grad wrt x
  void* dres;                 // backward: grad wrt residual (optional)
  int fp32;                   // 1: activations are float, 0: __nv_bfloat16
  const float* gamma;
  const float* beta;
  float* mean;                // saved batch mean   [C]
  float* invstd;              // saved 1/sqrt(var+eps)
  float* run_mean;            // optional running stats (updated in the stats kernel)
  float* run_var;
  long long* nbt;             // optional num_batches_tracked
  float* dgamma;              // backward outputs (fp32) -- also inputs of the dx kernel
  float* dbeta;
  float* partial;             // workspace [bn_partial_rows][128]
  unsigned int* ticket;       // [64]: per-slice tickets [0..31], global epoch ticket [63]
  unsigned int* flag;         // [32] per-slice epoch flags (fused kernels)
  unsigned int* epoch;        // [1]  launch epoch (device resident: graph-replay safe)
  int* status;                // sticky error word (2 = fused-kernel wait timed out)
  long long M;
  int C;
  float eps;
  float momentum;
  int relu;
  int fused_ok;               // allow the single-launch fused path when the grid is co-resident
  // fp32 only, optional: ALSO emit the result as three bf16 planes [3][M*C] (x = p0+p1+p2) -- the operand format of
  // the tensor-core convolutions (csrc/conv_tc.cu), so the consumer conv needs no separate split pass
  __nv_bfloat16* y_planes;    // forward: planes of y
  __nv_bfloat16* dx_planes;   // backward: planes of dx (= dY of the convolution that produced x)
  // ReLU mask of the backward (split kernels; BN_MASK_* in bn_common.cuh): 0 = y > 0 read from p.y; 1 = recomputed
  // from x as fmaf(x, sc, sh) > 0, bit for bit what the apply kernel decided (no residual only); 2 = the bit mask p.mask.
  // p.mask [M*C/8]: bit e of byte (row*C + c)/8 is the mask of channel c+e (c a multiple of 8); the forward apply
  // kernel writes it when non-null.  The backward skips the fp32 dx store when p.dx is null (planes only).
  int mask_mode;
  unsigned char* mask;
};
int bn_partial_rows(int sm_count);
// fp32 NCHW variant (csrc/bn_nchw.cu): `hw` = H*W (multiple of 4), p.M = N*H*W.  Workspace: p.partial >= C*64*2
// floats, p.ticket >= C words (p.flag / p.epoch unused).
cudaError_t launch_bn_nchw(const BnParams& p, int hw, int which, int sm_count, cudaStream_t s);
// which: 0 training forward, 1 apply only (eval), 2 backward
cudaError_t launch_bn(const BnParams& p, int which, int sm_count, cudaStream_t s);

// ------------------------------------------------------------------ wgmma fused Linear(+bias)(+ReLU)
// Y[M,N] = act(X[M,K] * W[N,K]^T + b): bf16 operands, fp32 accumulation in registers (csrc/linear_tc_tma.cu).
struct LinearParams {
  const __nv_bfloat16* x;   // [M, K] row-major
  const __nv_bfloat16* w;   // [N, K] row-major (nn.Linear weight layout)
  const float* bias;        // [N] or null
  void* y;                  // [M, N] bf16 or fp32
  int M, N, K;              // N % 16 == 0, 16 <= N <= 256, K % 8 == 0
  int relu;
  int out_bf16;
};
// TMA + SWIZZLE_128B + persistent CTAs (one per SM) + two wgmma warpgroups
cudaError_t launch_linear_tc_tma(const LinearParams& p, int sm_count, cudaStream_t s);

// ------------------------------------------------------------------ wgmma convolutions at fp32 accuracy
// (csrc/conv_tc.cu): fp32 tensors split into three bf16 planes, six bf16 MMAs per fp32 product, fp32 accumulation.
// One kernel pair + a tap table covers 3x3 stride 1/2, 1x1 stride 2 and the 3-channel stem (see conv_tc.cu).
struct ConvTcParams {
  const __nv_bfloat16* a;   // activation planes [3][nsrc][N][H][W][Ca] (forward: x; dgrad: dY; wgrad: x)
  const __nv_bfloat16* b;   // fprop/dgrad: weight planes [3][Cb][wtaps*Ca]; wgrad: dY planes [3][N][H][W][Cb]
  float* out;               // fprop/dgrad: [N][OH][OW][Cb]; wgrad: workspace [splits][ntaps*Ca][Cb]
  int N, H, W;              // pixel grid of the GEMM rows
  int Ca, Cb;
  int ntaps, nsrc, wtaps;   // taps of this launch, source sub-images per plane, taps in the weight matrix
  signed char dh[9], dw[9], src[9], wk[9];
  int OH, OW, os, op, oq;   // fprop: pixel (n,i,j) -> out[n][i*os+op][j*os+oq]
  float* dwout;             // wgrad: [Cb][ntaps*Ca] (OHWI); written directly by the kernel when there is one split
  float* ws;                // fprop: workspace [ksplits][m_tiles*128][Cb] when ksplits > 1
  int ksplits;              // fprop: K-loop splits (conv_fprop_ksplits(); 1 = none)
  int bh, bn, m_tiles, k_blocks;   // filled in by the launchers
  // fprop/dgrad, optional: out = acc + (mask bit ? addend : 0.f), addend [N][OH][OW][Cb] fp32 and addmask one bit per
  // element in the BnParams::mask layout -- the skip-connection gradient of an identity block, added in the epilogue
  // of its first convolution's data gradient
  const float* addend;
  const unsigned char* addmask;
};
bool conv_tc_supported(int N, int H, int W, int Ca, int Cb);
int conv_wgrad_splits(int N, int H, int W, int Ca, int Cb, int ntaps, int sm_count);
int conv_fprop_ksplits(int N, int H, int W, int Ca, int Cb, int ntaps, int sm_count);
int conv_fprop_mtiles(int N, int H, int W);   // 128-pixel tiles of the grid (workspace rows = 128 * this)
int conv_fprop_ntile(int N, int H, int W, int Ca, int Cb, int ntaps, int sm_count);   // N tile of the launch: 64 | 128
cudaError_t launch_conv_fprop(const ConvTcParams& p, int sm_count, cudaStream_t s);
cudaError_t launch_conv_wgrad(const ConvTcParams& p, float* dw, int splits, cudaStream_t s);
cudaError_t launch_split3(const float* src, __nv_bfloat16* dst, size_t n, cudaStream_t s);   // n % 8 == 0
cudaError_t launch_split3_parity(const float* src, __nv_bfloat16* dst, int N, int H, int W, int C, cudaStream_t s);
cudaError_t launch_split3_stem(const float* src, __nv_bfloat16* dst, int N, int H, int W, cudaStream_t s);
cudaError_t launch_conv_wprep(const float* w, __nv_bfloat16* wp, __nv_bfloat16* wtp, int Co, int T, int Ci, cudaStream_t s);
cudaError_t conv_graph_kernel_priorities(cudaGraph_t g, std::vector<std::pair<int, int>>* out);

// ------------------------------------------------------------------ IPC window runtime
// The RMA-window replacement (MPI_Alloc_mem + MPI_Win_create, event.cpp:138-147).
struct IpcHandle {
  unsigned char bytes[64];
};
cudaError_t ipc_alloc(size_t nbytes, void** ptr, IpcHandle* h);
cudaError_t ipc_open(const IpcHandle& h, void** ptr);
cudaError_t ipc_close(void* ptr);
cudaError_t ipc_free(void* ptr);

}  // namespace egb
