// eventgrad_b200 -- Python bindings (pybind11 + CUDA runtime only; no torch headers, so the
// whole extension rebuilds in seconds and carries no libtorch ABI coupling).  Tensors cross the
// boundary as raw device addresses (tensor.data_ptr()); streams as torch's cuda_stream handle.
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include <cstring>
#include <functional>
#include <stdexcept>
#include <string>
#include <tuple>
#include <type_traits>
#include <vector>
#include <unordered_map>

#include "api.h"
#include "host_loader.h"

namespace py = pybind11;
using namespace egb;

static void check(cudaError_t e, const char* what) {
  if (e != cudaSuccess) throw std::runtime_error(std::string(what) + ": " + cudaGetErrorString(e));
}

template <class S>
using Setter = std::function<void(S&, py::object)>;

#define PTRF(S, f) \
  { #f, [](S& p, py::object v) { p.f = reinterpret_cast<decltype(p.f)>(v.cast<uintptr_t>()); } }
#define NUMF(S, f) \
  { #f, [](S& p, py::object v) { p.f = v.cast<decltype(p.f)>(); } }
#define PTRF2(S, sub, f) \
  { #sub "." #f, [](S& p, py::object v) { p.sub.f = reinterpret_cast<decltype(p.sub.f)>(v.cast<uintptr_t>()); } }
#define NUMF2(S, sub, f) \
  { #sub "." #f, [](S& p, py::object v) { p.sub.f = v.cast<decltype(p.sub.f)>(); } }

// pointer array of EG_MAX_SLOTS entries from a Python list (missing entries are null)
#define ARRF(S, f)                                                                                       \
  {                                                                                                      \
    #f, [](S& p, py::object v) {                                                                         \
      const auto l = v.cast<std::vector<uintptr_t>>();                                                   \
      if (l.size() > EG_MAX_SLOTS) throw std::invalid_argument(#f ": more than EG_MAX_SLOTS entries");   \
      for (size_t i = 0; i < EG_MAX_SLOTS; ++i)                                                          \
        p.f[i] = reinterpret_cast<std::remove_reference_t<decltype(p.f[0])>>(i < l.size() ? l[i] : 0);   \
    }                                                                                                    \
  }

#define TAB_FIELDS(S)                                                                              \
  PTRF2(S, tab, tile_tensor), PTRF2(S, tab, t_tile_start), PTRF2(S, tab, t_tile_count),            \
      PTRF2(S, tab, t_numel), PTRF2(S, tab, t_msg_bytes), NUMF2(S, tab, n_tiles), NUMF2(S, tab, n_tensors)

static const std::unordered_map<std::string, Setter<GossipParams>> kGossip = {
    PTRF(GossipParams, theta), PTRF(GossipParams, grad), PTRF(GossipParams, mom),
    PTRF(GossipParams, inbox_l), PTRF(GossipParams, inbox_r), PTRF(GossipParams, push_l),
    PTRF(GossipParams, push_r), PTRF(GossipParams, shadow), PTRF(GossipParams, t_grad_ptr),
    PTRF(GossipParams, t_grad_bf16), PTRF(GossipParams, tile_ss),
    PTRF(GossipParams, tile_ss_l), PTRF(GossipParams, tile_ss_r), PTRF(GossipParams, flag_from_l),
    PTRF(GossipParams, flag_from_r), PTRF(GossipParams, flag_to_l), PTRF(GossipParams, flag_to_r),
    PTRF(GossipParams, ack_from_l), PTRF(GossipParams, ack_from_r), PTRF(GossipParams, ack_to_l),
    PTRF(GossipParams, ack_to_r), PTRF(GossipParams, pushed_from_l), PTRF(GossipParams, pushed_from_r),
    PTRF(GossipParams, pushed_to_l), PTRF(GossipParams, pushed_to_r), PTRF(GossipParams, ticket), PTRF(GossipParams, tensor_done), PTRF(GossipParams, status),
    NUMF(GossipParams, timeout_ns), NUMF(GossipParams, lr), NUMF(GossipParams, mu),
    NUMF(GossipParams, do_mix), NUMF(GossipParams, do_push), NUMF(GossipParams, sync),
    NUMF(GossipParams, send_ack), NUMF(GossipParams, zero_grad), NUMF(GossipParams, group_iters),
    PTRF(GossipParams, sparse), NUMF(GossipParams, need_norm), NUMF(GossipParams, phase), TAB_FIELDS(GossipParams),
    NUMF(GossipParams, wd), NUMF(GossipParams, nesterov), PTRF(GossipParams, lr_table), NUMF(GossipParams, lr_len),
    NUMF(GossipParams, local_steps), PTRF(GossipParams, sent), NUMF(GossipParams, global_avg_period),
    NUMF(GossipParams, quasi_global),
    PTRF2(GossipParams, fsm, thres), PTRF2(GossipParams, fsm, last_norm), PTRF2(GossipParams, fsm, last_iter),
    PTRF2(GossipParams, fsm, slopes), PTRF2(GossipParams, fsm, fire), PTRF2(GossipParams, fsm, cur_norm),
    PTRF2(GossipParams, fsm, counters), PTRF2(GossipParams, fsm, pass_num), PTRF2(GossipParams, fsm, log_ring),
    NUMF2(GossipParams, fsm, log_cap), NUMF2(GossipParams, fsm, horizon), NUMF2(GossipParams, fsm, constant),
    NUMF2(GossipParams, fsm, thres_type), NUMF2(GossipParams, fsm, history),
    NUMF2(GossipParams, fsm, initial_comm_passes), NUMF2(GossipParams, fsm, enabled),
    NUMF2(GossipParams, fsm, metric),
};

static const std::unordered_map<std::string, Setter<GraphSlots>> kGraph = {
    NUMF(GraphSlots, n_slots), NUMF(GraphSlots, period), ARRF(GraphSlots, inbox), ARRF(GraphSlots, push), ARRF(GraphSlots, flag_from),
    ARRF(GraphSlots, flag_to), ARRF(GraphSlots, ack_from), ARRF(GraphSlots, ack_to),
};

static const std::unordered_map<std::string, Setter<Q8Slots>> kQ8 = {
    PTRF(Q8Slots, q_from_l), PTRF(Q8Slots, q_from_r), PTRF(Q8Slots, s_from_l), PTRF(Q8Slots, s_from_r),
    PTRF(Q8Slots, q_to_l), PTRF(Q8Slots, q_to_r), PTRF(Q8Slots, s_to_l), PTRF(Q8Slots, s_to_r),
    PTRF(Q8Slots, prev), PTRF(Q8Slots, rep_l), PTRF(Q8Slots, rep_r), NUMF(Q8Slots, codec), NUMF(Q8Slots, gamma),
};

static const std::unordered_map<std::string, Setter<TrackSlots>> kTrack = {
    PTRF(TrackSlots, y), PTRF(TrackSlots, g_prev), PTRF(TrackSlots, y_in_l), PTRF(TrackSlots, y_in_r),
    PTRF(TrackSlots, y_to_l), PTRF(TrackSlots, y_to_r),
};

static const std::unordered_map<std::string, Setter<EdSlots>> kEd = {
    PTRF(EdSlots, psi),
};

static const std::unordered_map<std::string, Setter<MatchSlots>> kMatch = {
    NUMF(MatchSlots, world), NUMF(MatchSlots, rank), NUMF(MatchSlots, seed), PTRF(MatchSlots, peers),
    PTRF(MatchSlots, inbox), PTRF(MatchSlots, flag_from), PTRF(MatchSlots, done),
};

static const std::unordered_map<std::string, Setter<RoundParams>> kRounds = {
    PTRF(RoundParams, theta), PTRF(RoundParams, pass_num), PTRF(RoundParams, ticket), PTRF(RoundParams, status),
    NUMF(RoundParams, timeout_ns), NUMF(RoundParams, n_tiles), NUMF(RoundParams, group_iters),
    NUMF(RoundParams, rounds), NUMF(RoundParams, n_slots), ARRF(RoundParams, inbox), ARRF(RoundParams, push),
    ARRF(RoundParams, flag_from), ARRF(RoundParams, flag_to), ARRF(RoundParams, ack_from), ARRF(RoundParams, ack_to),
};

static const std::unordered_map<std::string, Setter<ChebParams>> kCheb = {
    PTRF(ChebParams, prev), PTRF(ChebParams, coef),
};

static const std::unordered_map<std::string, Setter<AllReduceParams>> kAllReduce = {
    PTRF(AllReduceParams, peer_bufs), PTRF(AllReduceParams, local), PTRF(AllReduceParams, theta),
    PTRF(AllReduceParams, mom), PTRF(AllReduceParams, shadow), PTRF(AllReduceParams, peer_flags),
    PTRF(AllReduceParams, flags), PTRF(AllReduceParams, ticket), PTRF(AllReduceParams, status),
    PTRF(AllReduceParams, step_ctr), NUMF(AllReduceParams, timeout_ns), NUMF(AllReduceParams, n_tiles),
    NUMF(AllReduceParams, rank), NUMF(AllReduceParams, world), NUMF(AllReduceParams, lr),
    NUMF(AllReduceParams, mu), NUMF(AllReduceParams, mode), NUMF(AllReduceParams, two_shot),
    NUMF(AllReduceParams, zero_after), PTRF(AllReduceParams, mc_local),
    NUMF(AllReduceParams, wd), NUMF(AllReduceParams, nesterov), PTRF(AllReduceParams, lr_table),
    NUMF(AllReduceParams, lr_len), PTRF(AllReduceParams, pass_num),
    PTRF(AllReduceParams, gate_pass), NUMF(AllReduceParams, gate_period),
};

// SlowMoParams: every AllReduceParams field plus the SlowMo block
static const std::unordered_map<std::string, Setter<SlowMoParams>> kSlowMo = [] {
  std::unordered_map<std::string, Setter<SlowMoParams>> m;
  for (const auto& kv : kAllReduce) {
    const Setter<AllReduceParams> f = kv.second;
    m.emplace(kv.first, [f](SlowMoParams& p, py::object v) { f(p, v); });
  }
  m.insert({PTRF(SlowMoParams, x), PTRF(SlowMoParams, u), NUMF(SlowMoParams, beta), NUMF(SlowMoParams, alpha)});
  return m;
}();

// ConsensusParams: every AllReduceParams field plus the table, the partial buffers and the ring
static const std::unordered_map<std::string, Setter<ConsensusParams>> kConsensus = [] {
  std::unordered_map<std::string, Setter<ConsensusParams>> m;
  for (const auto& kv : kAllReduce) {
    const Setter<AllReduceParams> f = kv.second;
    m.emplace(kv.first, [f](ConsensusParams& p, py::object v) { f(p, v); });
  }
  m.insert({PTRF(ConsensusParams, peer_part), PTRF(ConsensusParams, part), PTRF(ConsensusParams, tile_tensor),
            PTRF(ConsensusParams, t_tile_start), PTRF(ConsensusParams, t_tile_count), PTRF(ConsensusParams, t_numel),
            NUMF(ConsensusParams, n_tensors), PTRF(ConsensusParams, ring), PTRF(ConsensusParams, ring_step),
            PTRF(ConsensusParams, ring_ctr), NUMF(ConsensusParams, cap)});
  return m;
}();

static const std::unordered_map<std::string, Setter<SparseParams>> kSparse = {
    PTRF(SparseParams, theta), PTRF(SparseParams, prev), PTRF(SparseParams, rep_l), PTRF(SparseParams, rep_r),
    PTRF(SparseParams, rec_from_l), PTRF(SparseParams, rec_from_r), PTRF(SparseParams, rec_to_l),
    PTRF(SparseParams, rec_to_r), PTRF(SparseParams, seq_from_l), PTRF(SparseParams, seq_from_r),
    PTRF(SparseParams, seq_to_l), PTRF(SparseParams, seq_to_r), PTRF(SparseParams, applied_l),
    PTRF(SparseParams, applied_r), PTRF(SparseParams, done_from_l), PTRF(SparseParams, done_from_r),
    PTRF(SparseParams, done_to_l), PTRF(SparseParams, done_to_r), PTRF(SparseParams, ack_from_l),
    PTRF(SparseParams, ack_from_r), PTRF(SparseParams, ack_to_l), PTRF(SparseParams, ack_to_r),
    PTRF(SparseParams, t_k), PTRF(SparseParams, t_rec_off), PTRF(SparseParams, hist),
    PTRF(SparseParams, sel_prefix), PTRF(SparseParams, sel_remain), PTRF(SparseParams, cand),
    PTRF(SparseParams, cand_cnt), PTRF(SparseParams, done1), PTRF(SparseParams, done2), PTRF(SparseParams, desc),
    PTRF(SparseParams, bar), PTRF(SparseParams, fire),
    PTRF(SparseParams, pass_num), PTRF(SparseParams, ticket), PTRF(SparseParams, status),
    NUMF(SparseParams, timeout_ns), NUMF(SparseParams, sync), TAB_FIELDS(SparseParams),
};

static const std::unordered_map<std::string, Setter<BnParams>> kBn = {
    PTRF(BnParams, x), PTRF(BnParams, res), PTRF(BnParams, y), PTRF(BnParams, dy), PTRF(BnParams, dx),
    PTRF(BnParams, dres), PTRF(BnParams, gamma), PTRF(BnParams, beta), PTRF(BnParams, mean),
    PTRF(BnParams, invstd), PTRF(BnParams, run_mean), PTRF(BnParams, run_var), PTRF(BnParams, nbt),
    PTRF(BnParams, dgamma), PTRF(BnParams, dbeta), PTRF(BnParams, partial), PTRF(BnParams, ticket),
    PTRF(BnParams, flag), PTRF(BnParams, epoch), PTRF(BnParams, status), NUMF(BnParams, fused_ok),
    NUMF(BnParams, M), NUMF(BnParams, C), NUMF(BnParams, eps), NUMF(BnParams, momentum), NUMF(BnParams, relu),
    NUMF(BnParams, fp32),
};

template <class S>
static void bind_params(py::module_& m, const char* name, const std::unordered_map<std::string, Setter<S>>& tbl) {
  py::class_<S>(m, name)
      .def(py::init([]() {
        S p;
        std::memset(&p, 0, sizeof(S));
        return p;
      }))
      .def("set",
           [&tbl](S& p, const std::string& k, py::object v) {
             auto it = tbl.find(k);
             if (it == tbl.end()) throw std::invalid_argument("unknown field " + k);
             it->second(p, v);
           })
      .def("update",
           [&tbl](S& p, py::dict d) {
             for (auto kv : d) {
               const std::string k = kv.first.cast<std::string>();
               auto it = tbl.find(k);
               if (it == tbl.end()) throw std::invalid_argument("unknown field " + k);
               it->second(p, py::reinterpret_borrow<py::object>(kv.second));
             }
           })
      .def_static("fields", [&tbl]() {
        std::vector<std::string> v;
        for (auto& kv : tbl) v.push_back(kv.first);
        return v;
      });
}

static cudaStream_t S(uintptr_t s) { return reinterpret_cast<cudaStream_t>(s); }

// ---- launch accounting (api.h): relaxed atomics, one counter per kernel family
#include <atomic>
static std::atomic<long long> g_launches[egb::EG_FAM_N];
namespace egb {
void eg_count_launch(int family, int n) {
  if (family >= 0 && family < EG_FAM_N) g_launches[family].fetch_add(n, std::memory_order_relaxed);
}
}  // namespace egb

PYBIND11_MODULE(_C, m) {
  m.doc() = "eventgrad_b200 sm_90a kernels";
  m.attr("TILE") = EG_TILE;
  m.attr("arch") = "sm_90a";
  bind_params<GossipParams>(m, "GossipParams", kGossip);
  bind_params<GraphSlots>(m, "GraphSlots", kGraph);
  bind_params<Q8Slots>(m, "Q8Slots", kQ8);
  bind_params<TrackSlots>(m, "TrackSlots", kTrack);
  bind_params<EdSlots>(m, "EdSlots", kEd);
  bind_params<RoundParams>(m, "RoundParams", kRounds);
  bind_params<ChebParams>(m, "ChebParams", kCheb);
  bind_params<MatchSlots>(m, "MatchSlots", kMatch);
  m.attr("MATCH_PEER_BYTES") = (int)sizeof(MatchPeer);
  bind_params<AllReduceParams>(m, "AllReduceParams", kAllReduce);
  bind_params<SlowMoParams>(m, "SlowMoParams", kSlowMo);
  bind_params<ConsensusParams>(m, "ConsensusParams", kConsensus);
  bind_params<SparseParams>(m, "SparseParams", kSparse);
  bind_params<BnParams>(m, "BnParams", kBn);

  m.def("gossip_max_grid", &gossip_max_grid);
  m.def("gossip_step", [](const GossipParams& p, int grid, uintptr_t s) {
    check(launch_gossip_step(p, grid, S(s)), "gossip_step");
  });
  m.def("gossip_step_phase", [](GossipParams p, int phase, int grid, uintptr_t s) {
    p.phase = phase;
    check(launch_gossip_step(p, grid, S(s)), "gossip_step_phase");
  });
  m.def("ce_push", [](const GossipParams& p, uintptr_t s) { check(launch_ce_push(p, S(s)), "ce_push"); });
  m.def("gossip_dbuf_max_grid", &gossip_dbuf_max_grid);
  m.def("gossip_step_dbuf", [](const GossipParams& p, int grid, uintptr_t s) {
    check(launch_gossip_step_dbuf(p, grid, S(s)), "gossip_step_dbuf");
  });
  m.attr("MAX_SLOTS") = EG_MAX_SLOTS;
  m.def("gossip_graph_max_grid", &gossip_graph_max_grid);
  m.def("gossip_step_graph", [](const GossipParams& p, const GraphSlots& g, int grid, uintptr_t s) {
    check(launch_gossip_step_graph(p, g, grid, S(s)), "gossip_step_graph");
  });
  m.def("gossip_q8_max_grid", &gossip_q8_max_grid);
  m.def("gossip_step_q8", [](const GossipParams& p, const Q8Slots& q, int grid, uintptr_t s) {
    check(launch_gossip_step_q8(p, q, grid, S(s)), "gossip_step_q8");
  });
  m.def("gossip_gt_max_grid", &gossip_gt_max_grid);
  m.def("gossip_step_gt", [](const GossipParams& p, const TrackSlots& y, int grid, uintptr_t s) {
    check(launch_gossip_step_gt(p, y, grid, S(s)), "gossip_step_gt");
  });
  m.def("gossip_ed_max_grid", &gossip_ed_max_grid);
  m.def("gossip_step_ed", [](const GossipParams& p, const EdSlots& e, int grid, uintptr_t s) {
    check(launch_gossip_step_ed(p, e, grid, S(s)), "gossip_step_ed");
  });
  m.def("gossip_match_max_grid", &gossip_match_max_grid);
  m.def("gossip_step_match", [](const GossipParams& p, const MatchSlots& ms, int grid, uintptr_t s) {
    check(launch_gossip_step_match(p, ms, grid, S(s)), "gossip_step_match");
  });
  m.def("gossip_rounds_max_grid", &gossip_rounds_max_grid);
  m.def("gossip_rounds", [](const RoundParams& p, int grid, uintptr_t s) {
    check(launch_gossip_rounds(p, grid, S(s)), "gossip_rounds");
  });
  m.def("gossip_rounds_cheb", [](const RoundParams& p, const ChebParams& c, int grid, uintptr_t s) {
    check(launch_gossip_rounds_cheb(p, c, grid, S(s)), "gossip_rounds_cheb");
  });
  m.def("gossip_init", [](const GossipParams& p, int grid, int run_fsm, uintptr_t s) {
    check(launch_gossip_init(p, grid, run_fsm, S(s)), "gossip_init");
  });
  m.def("fsm_decide", [](const GossipParams& p, uintptr_t ext_norm, uintptr_t s) {
    check(launch_fsm_decide(p.fsm, p.tab, reinterpret_cast<const float*>(ext_norm), S(s)), "fsm_decide");
  });
  m.def("allreduce", [](const AllReduceParams& p, int grid, uintptr_t s) {
    check(launch_allreduce(p, grid, S(s)), "allreduce");
  });
  m.def("slowmo_sync", [](const SlowMoParams& p, int grid, uintptr_t s) {
    check(launch_slowmo_sync(p, grid, S(s)), "slowmo_sync");
  });
  m.def("consensus_max_grid", &consensus_max_grid);
  m.def("consensus", [](const ConsensusParams& p, int grid, uintptr_t s) {
    check(launch_consensus(p, grid, S(s)), "consensus");
  });
  m.def("allreduce_nvls", [](const AllReduceParams& p, int grid, uintptr_t s) {
    check(launch_allreduce_nvls(p, grid, S(s)), "allreduce_nvls");
  });
  m.def("sparse_select_push", [](const SparseParams& p, int grid, uintptr_t s) {
    check(launch_sparse_select_push(p, grid, S(s)), "sparse_select_push");
  });
  // device copy of a SparseParams block (GossipParams.sparse points at it: receive prologue of the mix kernel)
  m.attr("SPARSE_PARAMS_BYTES") = (int)sizeof(SparseParams);
  m.def("sparse_params_to_device", [](const SparseParams& p, uintptr_t dst) {
    check(cudaMemcpy(reinterpret_cast<void*>(dst), &p, sizeof(SparseParams), cudaMemcpyHostToDevice),
          "sparse_params_to_device");
  });
  m.def("sparse_apply", [](const SparseParams& p, int grid, uintptr_t s) {
    check(launch_sparse_apply(p, grid, S(s)), "sparse_apply");
  });
  m.def("launch_counts", []() {
    py::dict d;
    const char* names[egb::EG_FAM_N] = {"gossip", "allreduce", "sparse", "bn", "linear", "data", "conv"};
    for (int i = 0; i < egb::EG_FAM_N; ++i) d[names[i]] = g_launches[i].load(std::memory_order_relaxed);
    return d;
  });
  m.def("launch_count", []() {
    long long t = 0;
    for (int i = 0; i < egb::EG_FAM_N; ++i) t += g_launches[i].load(std::memory_order_relaxed);
    return t;
  });
  m.def("bn_partial_rows", &bn_partial_rows);
  m.def("bn_launch", [](const BnParams& p, int which, int sm_count, uintptr_t s) {
    check(launch_bn(p, which, sm_count, S(s)), "bn_launch");
  });
  // positional fast path (avoids the dict round trip on the per-layer hot path)
  // positional fast paths (no dict round trip on the per-layer hot path).  ws = {partial, ticket, flag,
  // epoch, status} device addresses of the shared workspace; `dir` 0 forward / 1 backward halves.
  m.def("bn_forward", [](uintptr_t x, uintptr_t res, uintptr_t y, uintptr_t gamma, uintptr_t beta, uintptr_t mean,
                         uintptr_t invstd, uintptr_t run_mean, uintptr_t run_var, uintptr_t nbt, uintptr_t partial,
                         uintptr_t ticket, uintptr_t flag, uintptr_t epoch, uintptr_t status, long long M, int C,
                         float eps, float momentum, int relu, int training, int fused_ok, int sm_count, int fp32,
                         int nchw_hw, uintptr_t s, uintptr_t y_planes, uintptr_t mask) {
    BnParams p;
    std::memset(&p, 0, sizeof(p));
    p.fp32 = fp32;
    p.x = reinterpret_cast<const void*>(x);
    p.res = reinterpret_cast<const void*>(res);
    p.y = reinterpret_cast<void*>(y);
    p.gamma = reinterpret_cast<const float*>(gamma);
    p.beta = reinterpret_cast<const float*>(beta);
    p.mean = reinterpret_cast<float*>(mean);
    p.invstd = reinterpret_cast<float*>(invstd);
    p.run_mean = reinterpret_cast<float*>(run_mean);
    p.run_var = reinterpret_cast<float*>(run_var);
    p.nbt = reinterpret_cast<long long*>(nbt);
    p.partial = reinterpret_cast<float*>(partial);
    p.ticket = reinterpret_cast<unsigned int*>(ticket);
    p.flag = reinterpret_cast<unsigned int*>(flag);
    p.epoch = reinterpret_cast<unsigned int*>(epoch);
    p.status = reinterpret_cast<int*>(status);
    p.M = M; p.C = C; p.eps = eps; p.momentum = momentum; p.relu = relu; p.fused_ok = fused_ok;
    if (y_planes != 0 && (!fp32 || nchw_hw > 0)) throw std::invalid_argument("bn_forward: planes need the fp32 NHWC path");
    p.y_planes = reinterpret_cast<__nv_bfloat16*>(y_planes);
    if (mask != 0 && (nchw_hw > 0 || !training)) throw std::invalid_argument("bn_forward: the bit mask needs the NHWC training path");
    p.mask = reinterpret_cast<unsigned char*>(mask);
    if (nchw_hw > 0)
      check(launch_bn_nchw(p, nchw_hw, training ? 0 : 1, sm_count, S(s)), "bn_forward (nchw)");
    else
      check(launch_bn(p, training ? 0 : 1, sm_count, S(s)), "bn_forward");
  });
  // mask_mode: BN_MASK_Y (read y) | BN_MASK_X (recompute from x, needs beta) | BN_MASK_BITS (read `mask`); dx may be 0
  // when dx_planes is given
  m.def("bn_backward", [](uintptr_t x, uintptr_t y, uintptr_t dy, uintptr_t dx, uintptr_t dres, uintptr_t gamma,
                          uintptr_t mean, uintptr_t invstd, uintptr_t dgamma, uintptr_t dbeta, uintptr_t partial,
                          uintptr_t ticket, uintptr_t flag, uintptr_t epoch, uintptr_t status, long long M, int C,
                          int relu, int fused_ok, int sm_count, int fp32, int nchw_hw, uintptr_t s,
                          uintptr_t dx_planes, uintptr_t beta, int mask_mode, uintptr_t mask) {
    BnParams p;
    std::memset(&p, 0, sizeof(p));
    p.fp32 = fp32;
    p.x = reinterpret_cast<const void*>(x);
    p.y = reinterpret_cast<void*>(y);
    p.dy = reinterpret_cast<const void*>(dy);
    p.dx = reinterpret_cast<void*>(dx);
    p.dres = reinterpret_cast<void*>(dres);
    p.gamma = reinterpret_cast<const float*>(gamma);
    p.mean = reinterpret_cast<float*>(mean);
    p.invstd = reinterpret_cast<float*>(invstd);
    p.dgamma = reinterpret_cast<float*>(dgamma);
    p.dbeta = reinterpret_cast<float*>(dbeta);
    p.partial = reinterpret_cast<float*>(partial);
    p.ticket = reinterpret_cast<unsigned int*>(ticket);
    p.flag = reinterpret_cast<unsigned int*>(flag);
    p.epoch = reinterpret_cast<unsigned int*>(epoch);
    p.status = reinterpret_cast<int*>(status);
    p.M = M; p.C = C; p.relu = relu; p.fused_ok = fused_ok;
    if (dx_planes != 0 && (!fp32 || nchw_hw > 0)) throw std::invalid_argument("bn_backward: planes need the fp32 NHWC path");
    p.dx_planes = reinterpret_cast<__nv_bfloat16*>(dx_planes);
    p.beta = reinterpret_cast<const float*>(beta);
    p.mask_mode = mask_mode;
    p.mask = reinterpret_cast<unsigned char*>(mask);
    if (mask_mode < 0 || mask_mode > 2 || (mask_mode == 1 && beta == 0) || (mask_mode == 2 && mask == 0) ||
        (mask_mode != 0 && (nchw_hw > 0 || !fp32)) || (dx == 0 && dx_planes == 0))
      throw std::invalid_argument("bn_backward: bad mask source / outputs");
    if (nchw_hw > 0)
      check(launch_bn_nchw(p, nchw_hw, 2, sm_count, S(s)), "bn_backward (nchw)");
    else
      check(launch_bn(p, 2, sm_count, S(s)), "bn_backward");
  });
  m.def("linear_tc", [](uintptr_t x, uintptr_t w, uintptr_t bias, uintptr_t y, int M, int N, int K, int relu,
                            int out_bf16, int sm_count, uintptr_t s) {
    LinearParams p;
    p.x = reinterpret_cast<const __nv_bfloat16*>(x);
    p.w = reinterpret_cast<const __nv_bfloat16*>(w);
    p.bias = reinterpret_cast<const float*>(bias);
    p.y = reinterpret_cast<void*>(y);
    p.M = M; p.N = N; p.K = K; p.relu = relu; p.out_bf16 = out_bf16;
    check(launch_linear_tc_tma(p, sm_count, S(s)), "linear_tc");
  });
  m.def("conv_tc_supported", [](int N, int H, int W, int Ca, int Cb) { return conv_tc_supported(N, H, W, Ca, Cb); });
  m.def("conv_wgrad_splits", [](int N, int H, int W, int Ca, int Cb, int ntaps, int sm) {
    return conv_wgrad_splits(N, H, W, Ca, Cb, ntaps, sm);
  });
  m.def("conv_fprop_ksplits", [](int N, int H, int W, int Ca, int Cb, int ntaps, int sm) {
    return conv_fprop_ksplits(N, H, W, Ca, Cb, ntaps, sm);
  });
  m.def("conv_fprop_mtiles", [](int N, int H, int W) { return conv_fprop_mtiles(N, H, W); });
  m.def("conv_fprop_ntile", [](int N, int H, int W, int Ca, int Cb, int ntaps, int sm) {
    return conv_fprop_ntile(N, H, W, Ca, Cb, ntaps, sm);
  });
  m.def("split3", [](uintptr_t src, uintptr_t dst, size_t n, uintptr_t s) {
    check(launch_split3(reinterpret_cast<const float*>(src), reinterpret_cast<__nv_bfloat16*>(dst), n, S(s)), "split3");
  });
  m.def("split3_parity", [](uintptr_t src, uintptr_t dst, int N, int H, int W, int C, uintptr_t s) {
    check(launch_split3_parity(reinterpret_cast<const float*>(src), reinterpret_cast<__nv_bfloat16*>(dst), N, H, W, C, S(s)),
          "split3_parity");
  });
  m.def("split3_stem", [](uintptr_t src, uintptr_t dst, int N, int H, int W, uintptr_t s) {
    check(launch_split3_stem(reinterpret_cast<const float*>(src), reinterpret_cast<__nv_bfloat16*>(dst), N, H, W, S(s)),
          "split3_stem");
  });
  m.def("conv_wprep", [](uintptr_t w, uintptr_t wp, uintptr_t wtp, int Co, int T, int Ci, uintptr_t s) {
    check(launch_conv_wprep(reinterpret_cast<const float*>(w), reinterpret_cast<__nv_bfloat16*>(wp),
                            reinterpret_cast<__nv_bfloat16*>(wtp), Co, T, Ci, S(s)), "conv_wprep");
  });
  // taps: list of (dh, dw, src, wk)
  auto fill = [](ConvTcParams& p, const std::vector<std::tuple<int, int, int, int>>& taps) {
    if (taps.empty() || taps.size() > 9) throw std::invalid_argument("1..9 taps");
    p.ntaps = (int)taps.size();
    for (int t = 0; t < p.ntaps; ++t) {
      p.dh[t] = (signed char)std::get<0>(taps[t]);
      p.dw[t] = (signed char)std::get<1>(taps[t]);
      p.src[t] = (signed char)std::get<2>(taps[t]);
      p.wk[t] = (signed char)std::get<3>(taps[t]);
    }
  };
  m.def("conv_fprop", [fill](uintptr_t a, uintptr_t b, uintptr_t out, int N, int H, int W, int Ca, int Cb,
                             std::vector<std::tuple<int, int, int, int>> taps, int nsrc, int wtaps, int OH, int OW, int os,
                             int op, int oq, int sm_count, uintptr_t s, uintptr_t ws, int ksplits, uintptr_t addend,
                             uintptr_t addmask) {
    ConvTcParams p{};
    p.a = reinterpret_cast<const __nv_bfloat16*>(a);
    p.b = reinterpret_cast<const __nv_bfloat16*>(b);
    p.out = reinterpret_cast<float*>(out);
    p.N = N; p.H = H; p.W = W; p.Ca = Ca; p.Cb = Cb; p.nsrc = nsrc; p.wtaps = wtaps;
    p.OH = OH; p.OW = OW; p.os = os; p.op = op; p.oq = oq;
    p.ws = reinterpret_cast<float*>(ws); p.ksplits = ksplits;
    if ((addend == 0) != (addmask == 0)) throw std::invalid_argument("conv_fprop: addend and addmask go together");
    p.addend = reinterpret_cast<const float*>(addend);
    p.addmask = reinterpret_cast<const unsigned char*>(addmask);
    fill(p, taps);
    check(launch_conv_fprop(p, sm_count, S(s)), "conv_fprop");
  });
  m.def("conv_wgrad", [fill](uintptr_t x, uintptr_t g, uintptr_t ws, uintptr_t dw, int N, int H, int W, int Ca, int Cb,
                             std::vector<std::tuple<int, int, int, int>> taps, int nsrc, int splits, uintptr_t s) {
    ConvTcParams p{};
    p.a = reinterpret_cast<const __nv_bfloat16*>(x);
    p.b = reinterpret_cast<const __nv_bfloat16*>(g);
    p.out = reinterpret_cast<float*>(ws);
    p.N = N; p.H = H; p.W = W; p.Ca = Ca; p.Cb = Cb; p.nsrc = nsrc; p.wtaps = (int)taps.size();
    p.OH = H; p.OW = W; p.os = 1;
    fill(p, taps);
    check(launch_conv_wgrad(p, reinterpret_cast<float*>(dw), splits, S(s)), "conv_wgrad");
  });
  m.def("conv_graph_kernel_priorities", [](uintptr_t graph) {
    std::vector<std::pair<int, int>> out;
    check(conv_graph_kernel_priorities(reinterpret_cast<cudaGraph_t>(graph), &out), "conv_graph_kernel_priorities");
    return out;
  });
  m.def("decode_augment",
        [](uintptr_t in, uintptr_t out, uintptr_t oy, uintptr_t ox, uintptr_t flip, int B, int C, int H, int W,
           int pad, float scale, float mean, float inv_std, int out_bf16, int nhwc, uintptr_t s) {
          check(launch_decode_augment(reinterpret_cast<const uint8_t*>(in), reinterpret_cast<void*>(out),
                                      reinterpret_cast<const int*>(oy), reinterpret_cast<const int*>(ox),
                                      reinterpret_cast<const int*>(flip), B, C, H, W, pad, scale, mean,
                                      inv_std, out_bf16, nhwc, S(s)),
                "decode_augment");
        });

  // ---- native host-side batch prefetcher (data/native_loader.py) --------------------------------
  py::class_<HostPrefetcher>(m, "HostPrefetcher")
      .def(py::init([](uintptr_t images, uintptr_t labels, int64_t n, int64_t sample_bytes, int64_t batch,
                       std::vector<uintptr_t> slot_images, std::vector<uintptr_t> slot_labels) {
        if (slot_images.size() != slot_labels.size() || slot_images.empty())
          throw std::invalid_argument("need the same positive number of image and label slots");
        std::vector<uint8_t*> si;
        std::vector<int64_t*> sl;
        for (auto p : slot_images) si.push_back(reinterpret_cast<uint8_t*>(p));
        for (auto p : slot_labels) sl.push_back(reinterpret_cast<int64_t*>(p));
        return new HostPrefetcher(reinterpret_cast<const uint8_t*>(images), reinterpret_cast<const int64_t*>(labels), n,
                                  sample_bytes, batch, std::move(si), std::move(sl));
      }))
      .def("start_epoch", [](HostPrefetcher& h, uintptr_t order, int64_t n_order) {
        h.start_epoch(reinterpret_cast<const int64_t*>(order), n_order);
      })
      .def("num_batches", &HostPrefetcher::num_batches)
      .def("next", [](HostPrefetcher& h) {
        std::pair<int, int64_t> r;
        {
          py::gil_scoped_release nogil;      // the worker thread never needs the GIL; do not hold it while waiting
          r = h.next();
        }
        return py::make_tuple(r.first, r.second);
      })
      .def("release", &HostPrefetcher::release)
      .def("stop", &HostPrefetcher::stop);

  // ---- IPC window runtime -------------------------------------------------------------------
  m.def("ipc_alloc", [](size_t nbytes) {
    void* ptr = nullptr;
    IpcHandle h;
    check(ipc_alloc(nbytes, &ptr, &h), "ipc_alloc");
    return py::make_tuple(reinterpret_cast<uintptr_t>(ptr),
                          py::bytes(reinterpret_cast<const char*>(h.bytes), sizeof(h.bytes)));
  });
  m.def("ipc_open", [](py::bytes hb) {
    std::string s = hb;
    if (s.size() != sizeof(IpcHandle)) throw std::invalid_argument("bad IPC handle size");
    IpcHandle h;
    std::memcpy(h.bytes, s.data(), sizeof(h.bytes));
    void* ptr = nullptr;
    check(ipc_open(h, &ptr), "ipc_open");
    return reinterpret_cast<uintptr_t>(ptr);
  });
  m.def("ipc_close", [](uintptr_t p) { check(ipc_close(reinterpret_cast<void*>(p)), "ipc_close"); });
  m.def("ipc_free", [](uintptr_t p) { check(ipc_free(reinterpret_cast<void*>(p)), "ipc_free"); });
  m.def("device_can_access_peer", [](int dev, int peer) {
    int ok = 0;
    check(cudaDeviceCanAccessPeer(&ok, dev, peer), "cudaDeviceCanAccessPeer");
    return ok != 0;
  });
}
