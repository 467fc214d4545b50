// net.cuh — the Q-network object: fp32 master weights (online + target), RMSProp state,
// activations, gradient partials, all resident in HBM.
#pragma once
#include <cuda_fp16.h>

#include "common.cuh"
#include "net_simt.cuh"
#include "replay.cuh"
#include "comm_p2p.cuh"
#include "optim.cuh"

namespace b200 {

constexpr int kLayers = 5;
constexpr int kMaxActions = 32;
constexpr int kMaxAtoms = 64;             // distributional head: atoms per action
constexpr int kMaxQuantiles = 200;        // quantile-regression head: quantiles per action
constexpr int kMaxRemHeads = 200;         // random ensemble mixture head: heads per action
constexpr int kCostRing = 1024;
constexpr int kHostCosts = 60;            // per-step costs mirrored in host-mapped memory
constexpr int kHostQ = 64, kHostQFloats = 960;   // word offset / capacity of the Q rows in the host-mapped block
constexpr int kFc1Splits = 14;            // 3136 / 14 = 224 = 14 * 16
constexpr int kFc1Chunk = kFlat / kFc1Splits;
constexpr int kIqnWgradRows = 256;
constexpr int kMaxCropPad = 8;            // random-shift augmentation: pads 1..8        // IQN on the tensor-core engine: expanded rows per fc1 wgrad partial

struct LayerTable {
  int64_t off[kLayers + 1];   // element offsets into the all-layer parameter vector
  int rows[kLayers], cols[kLayers];  // internal [K][N] shape
  int64_t part_off[kLayers];  // element offsets into the split-K partial scratch
  int splits[kLayers];
};

// What a captured CUDA graph was captured at: a step graph at a ring, a predict graph at a state window and row count.
// A graph is stale as soon as one field differs.
struct GraphKey {
  const void* src = nullptr;   // the ring (a step) or the device-resident state window (predict)
  uint64_t serial = 0;         // b200dqn_replay::serial: the pointer alone can name a newer ring
  cudaStream_t stream = nullptr;
  int world = 0, trace_gen = 0, rows = 0;
  uint32_t per_gen = 0;        // b200dqn_replay::per_gen
  int nstep = 1;               // b200dqn_replay::nstep
  bool operator==(const GraphKey& o) const {
    return src == o.src && serial == o.serial && stream == o.stream && world == o.world && trace_gen == o.trace_gen &&
           rows == o.rows && per_gen == o.per_gen && nstep == o.nstep;
  }
};

struct GraphCache {
  cudaGraphExec_t exec = nullptr;
  GraphKey key{};
  void drop() {
    if (exec) { cudaGraphExecDestroy(exec); exec = nullptr; }
  }
};

}  // namespace b200

struct b200dqn_net {
  int device = 0;
  int sm_count = 132;      // queried at create; sizes the capped elementwise grids
  b200dqn_net_config cfg{};
  int nb = 0;  // per-rank minibatch
  int A = 0;
  b200::LayerTable lt{};
  int64_t n_params = 0;

  // parameters (internal layout, all layers contiguous)
  float* d_w = nullptr;   // online weights
  float* d_s = nullptr;   // online optimizer state: n_states planes of n_params (RMSProp 1, Adam 2, Adadelta 3)
  int n_states = 1;
  float* d_optscal = nullptr;  // [0] Adam's step scalar l of the current step (written by the head kernel);
                               // [1] (as u32) fast-path predicts completed
  uint32_t* d_optscal_u32() const { return reinterpret_cast<uint32_t*>(d_optscal) + 1; }
  float* d_tw = nullptr;  // target weights (== d_w when target_steps == 0)
  float* d_ts = nullptr;  // target optimizer state (copied for fidelity with :102-105)
  float* d_g = nullptr;   // summed gradients (all-reduce buffer / get_grads)
  float* d_part = nullptr;  // split-K partials
  int64_t part_elems = 0;

  // activations: [0] online, [1] target, [2] online on the poststates (Double DQN; SIMT engine only, allocated
  // when double Q is first switched on)
  float* d_h1[3] = {}, *d_h2[3] = {}, *d_h3[3] = {}, *d_h4[2] = {};
  float* d_fc1part = nullptr;  // [2*splits][nb][hidden], [3*splits][nb][hidden] once double Q has been switched on
  float* d_q[3] = {};          // [nb][A]: preq, postq, Q_online_post (Double DQN)
  float* d_delta = nullptr;    // [nb][A] clipped
  float* d_dz4 = nullptr, *d_dz3 = nullptr, *d_dz2 = nullptr, *d_dz1 = nullptr;
  float* d_cost = nullptr;     // cost ring [kCostRing]
  uint32_t* d_step = nullptr;  // device step counter (cost ring cursor)
  float* d_rowcost = nullptr;    // [nb] per-sample cost
  // host-mapped result block (4 KB): [0] train steps completed (published last, after a system fence), [1]
  // action-range flag, [2] predicts completed, [4 + (step % kHostCosts)] cost of that step (k_cost_finish);
  // [64 ..) Q rows of the last fast-path predict (k_publish_q)
  volatile uint32_t* h_res = nullptr;
  uint32_t predicts_launched = 0;
  b200::GraphCache graph_predict;   // forward on a device-resident state window + result publish
  b200dqn_replay* step_replay = nullptr;   // set while a step that samples from a ring is being enqueued / captured

  // unfused-mode staging (host minibatch -> device)
  uint8_t* d_pre = nullptr, *d_post = nullptr, *d_act = nullptr, *d_term = nullptr;
  int64_t* d_rew = nullptr;
  int32_t* d_iota1 = nullptr;  // b
  int32_t* d_iota4 = nullptr;  // hist * b
  uint8_t* h_pin = nullptr;    // pinned staging for predict/train host entry points
  size_t pin_bytes = 0;

  int64_t train_iterations = 0;

  // step scheduling: side streams / events for the independent wgrad + optimizer branches, and the
  // captured CUDA graph of one fused step
  cudaStream_t side[4] = {};   // three wgrad/optimizer branches + the collective stream
  cudaEvent_t ev[19] = {};   // [15] / [16]: fork / join of the Munchausen target pass, of the IQN tau branch or of the
                             // REM mixture draw (a net has at most one of them); [17] / [18]: of the random-shift draw
  bool use_graph = true, use_branches = true;
  bool keep_grads = false;   // tensor-core dgrads also write the fp32 dZ3/dZ2/dZ1 (tests)
  bool double_q = false;     // Double DQN target: the online net picks the poststate action, the target net values it
  bool double_q_alloc = false;   // the third network slot's buffers exist
  b200::GraphCache graph_step;    // the fused step (sampler + train step)
  int graph_launches = 0;         // kernels launched by one captured fused step
  b200::GraphCache graph_train;   // same step without the sampler (train on pre-sampled indexes)
  int ring_nstep = 1;   // n-step length of the ring this net last trained from (comm_init refuses N > 1)
  float* d_td_err = nullptr;   // [nb] TD errors before the clip (prioritized replay; allocated at its first step)

  // distributional head (cfg.num_atoms > 0; nothing below is allocated otherwise).  fc2 has A * atoms outputs, and its
  // per-row gradient partials in d_part are compact: [nb][512][atoms], the taken action's block only.
  int atoms = 0;
  double dz = 0.0;               // (v_max - v_min) / (atoms - 1)
  float* d_logits = nullptr;     // [3][nb][A * atoms]
  float* d_probs = nullptr;      // [3][nb][A][atoms]
  float* d_tdist = nullptr;      // [nb][atoms] projected target distribution
  float* d_lgrad = nullptr;      // [nb][atoms] gradient on the taken action's logits
  int32_t* d_act_rows = nullptr; // [nb] taken action of each row of the last train step (selects the dW5 block)

  // quantile-regression head (cfg.num_quantiles > 0; nothing below is allocated otherwise).  fc2 has A * quantiles
  // outputs and shares the distributional head's compact dW5 partials, d_act_rows and fc2 kernels.
  int quantiles = 0;
  float* d_theta = nullptr;      // [3][nb][A * quantiles]
  float* d_tquant = nullptr;     // [nb][quantiles] target quantiles
  float* d_qgrad = nullptr;      // [nb][quantiles] gradient on the taken action's quantiles
  // random ensemble mixture head (cfg.num_heads > 0; nothing below is allocated otherwise).  fc2 has A * rem_k outputs,
  // theta in d_theta, and shares the distributional head's compact dW5 partials, d_act_rows and fc2 kernels
  int rem_k = 0;                             // K
  unsigned long long* d_rem_ctr = nullptr;   // the mixture's draw counter
  float* d_rem_alpha = nullptr;              // [K] the mixture alpha of the last train step
  float* d_rem_grad = nullptr;               // [nb][K] gradient on the taken action's heads
  // bootstrapped heads (cfg.bootstrap_heads > 0): the REM head's K-headed fc2 (rem_k = K, d_theta, d_rem_grad, the fc2
  // kernels) trained by k_head_boot; the mixture's counter and alpha are not allocated.  Nothing below is otherwise.
  bool boot = false;
  uint8_t* d_boot_mask = nullptr;            // [nb][K] bootstrap masks of the last train step
  float* d_boot_y = nullptr;                 // [nb][K] per-head targets float(y_k)
  float* d_boot_delta = nullptr;             // [nb][K] per-head TD errors delta_k
  int32_t* d_boot_head = nullptr;            // the head predict acts on (-1: the mean over the heads)
  // fc2 outputs per action of a per-action head (C51 atoms, QR quantiles or REM heads), 0 on the scalar and dueling
  // heads: such an fc2 is summed and updated by k_opt_fc2_dist from the compact [nb][512][block] partials
  int fc2_block() const { return atoms ? atoms : quantiles ? quantiles : iqn_n ? 1 : rem_k; }
  int fc2_cols() const { return fc2_block() ? A * fc2_block() : dueling ? A + 1 : A; }

  // dueling network (cfg.dueling): fc1 is kDuelHidden wide (advantage units [0, 512), value units [512, 1024)) and
  // fc2 is block-structured [512][A + 1]: column a < A reads the advantage units, column A the value units
  bool dueling = false;
  int hidden = b200::kHidden;    // fc1's width: H4, dZ4 and the fc1 partials are [.][hidden]
  float* d_va = nullptr;         // [3][nb][A + 1]: the advantages, then V, of every slot of the last forward

  // Munchausen target (cfg.munchausen): with a separate target network the train step runs it on the prestates as a
  // one-slot forward pass into the third slot's buffers (made at creation; Double DQN, their other user, is refused),
  // and the head reads its Q row as slot 2 (Q_TARGET_PRE = d_q[2])
  bool munchausen = false;
  float* d_tdtarget = nullptr;   // [nb] float(y) of the last train step

  // implicit quantile network head (cfg.num_tau_samples > 0; nothing below is allocated otherwise).  fc1 and fc2 run
  // on the expanded rows r = b N + j (b K + k on predict): H4, dZ4, the fc1 partials and fc2's per-row partials (block
  // width 1, summed by k_opt_fc2_dist) are sized by iqn_rows; the conv trunk runs at nb rows.
  int iqn_n = 0, iqn_k = 0;      // N, K
  int iqn_rows = 0;              // nb max(N, K)
  float* d_we = nullptr;         // online embedding [64][3136] (internal column order); d_wes: its n_states planes
  float* d_wes = nullptr;
  float* d_twe = nullptr;        // target embedding and states (== d_we / d_wes when target_steps == 0)
  float* d_twes = nullptr;
  float* d_weg = nullptr;        // dWe of the last train step
  unsigned long long* d_tau_ctr = nullptr;   // the draw counter
  float* d_tau = nullptr;        // [2][iqn_rows]
  float* d_cos = nullptr;        // [2][iqn_rows][64]
  float* d_phi = nullptr;        // [2][iqn_rows][3136]
  float* d_x = nullptr;          // [2][iqn_rows][3136]
  float* d_iqn_theta = nullptr;  // [2][iqn_rows][A]
  float* d_iqn_tq = nullptr;     // [nb][N]
  float* d_iqn_qgrad = nullptr;  // [nb N]
  float* d_dx = nullptr;         // [iqn_rows][3136]
  float* d_dphi = nullptr;       // [iqn_rows][3136]
  __half* d_x16 = nullptr;       // tensor-core engine: fp16 planes of X, per slot [hi iqn_rows x 3136 | lo]
  // rows one fc1 / fc2 pass runs at for `rows` samples: rows N in a train step, rows K on predict
  int expanded(int rows, bool train) const { return iqn_n ? rows * (train ? iqn_n : iqn_k) : rows; }

  // fully parameterized quantile function head (cfg.num_fractions > 0): an IQN net (iqn_n = iqn_k = N) whose tau is the
  // fraction proposal tauhat instead of a draw (d_tau_ctr stays unallocated), plus the fraction layer and the boundary
  // pass at tau_1..tau_{N-1}, which runs phi, X, fc1 and fc2 on buffers of its own (nb (N - 1) rows)
  int fqf_n = 0;                 // N
  float* d_wf = nullptr;         // online fraction layer [N][3136] (internal column order); d_wfs: its n_states planes
  float* d_wfs = nullptr;
  float* d_twf = nullptr;        // target fraction layer and states (== d_wf / d_wfs when target_steps == 0)
  float* d_twfs = nullptr;
  float* d_wfg = nullptr;        // dW_f of the last train step
  float* d_fl = nullptr;         // [nb][N] logits l
  float* d_fq = nullptr;         // [nb][N] proposal q
  float* d_ftau = nullptr;       // [nb][N + 1] fractions tau
  float* d_fg = nullptr;         // [nb][N - 1] fraction gradient g
  float* d_fdl = nullptr;        // [nb][N] logit gradient dl
  float* d_btau = nullptr;       // boundary pass, rows nb (N - 1): tau_1..tau_{N-1}, c, phi, X, H4, theta_bnd
  float* d_bcos = nullptr;
  float* d_bphi = nullptr;
  float* d_bx = nullptr;
  float* d_bh4 = nullptr;
  float* d_btheta = nullptr;
  __half* d_bx16 = nullptr;      // tensor-core engine: fp16 planes of the boundary X [hi | lo]

  // random-shift augmentation (cfg.random_shift > 0; nothing below is allocated otherwise): every train step draws
  // crop offsets on the device and conv1 reads its frames through them
  int crop_pad = 0;                       // p
  unsigned long long* d_crop_ctr = nullptr;   // the draw counter
  int32_t* d_crop = nullptr;              // [2][nb][2] (dy, dx) of the last train step: prestates, then poststates
  bool crop_forked = false;               // the step's draw was launched on its own branch (ev[17] / ev[18])

  // soft target update (cfg.soft_target_tau > 0): every train step blends the target towards the online network with
  // these factors, c = float(1 - tau), t = float(tau)
  bool soft = false;
  float soft_c = 1.f, soft_t = 0.f;

  // global gradient-norm clipping (cfg.max_grad_norm > 0): d_clip holds S_0..S_5 (f64), N (f64), c32 (f32 in slot 7),
  // then k_grad_sq's per-CTA partial sums, layer l's (5: the IQN / FQF embedding) from slot 8 + sq_base[l]
  bool clip = false;
  double* d_clip = nullptr;
  int64_t sq_base[7] = {};
  float* d_clip_c() const { return reinterpret_cast<float*>(d_clip + 7); }

  void* umma_state = nullptr;  // tensor-core engine: fp16 operand planes + weight tile images (net_umma.cu)

  // multi-GPU
  void* nccl_comm = nullptr;
  int rank = 0, world = 1;
  // peer-memory gradient exchange (comm_p2p.cuh): d_g and its flag words as mapped from every rank
  bool xchg_ok = false;
  int xchg_flags = 0;             // k_xchg switches (comm_p2p.cuh), B200DQN_XCHG_FLAGS
  int xchg_blocks = 0;            // CTA cap per exchange (0 = kXMaxBlocks), B200DQN_XCHG_BLOCKS
  int xchg_sched = 2;             // 2: gather fc1's operands + LL all-reduce of the small layers (default),
                                  // 1: two-shot exchange per layer, 0: two-shot, two collectives
  float* xg[8] = {};              // [rank] = d_g
  uint32_t* xflags[8] = {};       // [rank] = d_xflags (tail of the d_g allocation)
  void* xopened[8] = {};          // cudaIpcOpenMemHandle results to close
  uint32_t* d_xflags = nullptr;   // flag words written by the peers
  uint32_t* d_xepoch = nullptr;   // local epoch counters [channel][block]
  uint32_t* d_xerr = nullptr;     // sticky "a wait timed out" word
  // gather / LL exchange: a second peer-mapped allocation, sized at comm_init for the world
  //   [push flags 4 KB][LL lines: parity x source x lines][H3 gather: parity x (hi | lo)][dZ4 gather: same]
  uint8_t* d_xbuf = nullptr;
  uint8_t* xbuf[8] = {};          // [rank] = d_xbuf
  void* xbuf_opened[8] = {};
  int64_t x_ll_off = 0, x_ll_lines = 0;               // bytes; LL lines per (parity, source)
  int64_t x_h3_off = 0, x_h3_parity = 0, x_h3_lo = 0;   // bytes; bytes per parity; lo plane offset in elements
  int64_t x_dz_off = 0, x_dz_parity = 0, x_dz_lo = 0;
  int64_t x_dzll_off = 0, x_dzll_lines = 0;           // LL line area of the dZ4 gather: bytes; lines per (parity, source)
  uint32_t* d_xll_epoch = nullptr;   // [kXChannels] epochs, then [kXChannels] tickets (LL exchange)
  uint32_t* d_xpush_epoch = nullptr; // [kXPushChannels] epochs, then tickets (plane push)
};
