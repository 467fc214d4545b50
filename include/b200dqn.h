/*
 * b200dqn.h — C-ABI of libb200dqn.so: the H100-native (sm_90a) replay-and-train hot path
 * behind tambetm/simple_dqn's ReplayMemory / DeepQNetwork / StateBuffer call surface.
 *
 * The reference has no FFI of its own (it is pure Python calling Neon); the boundary is the
 * three Python classes constructed at /root/reference/src/main.py:103-105 and
 * /root/reference/src/agent.py:12.  Each entry point below names the reference interface it
 * replaces (file:line under /root/reference).  A maintainer binds them with ctypes — see
 * INTEGRATION.md for the stub.
 *
 * Conventions
 *   - every function returns 0 on success or a negative B200DQN_E* code; the message for the
 *     calling thread's last failure is b200dqn_last_error().
 *   - plain pointers and sizes only.  `stream` is a cudaStream_t passed as void* (NULL = the
 *     legacy default stream).  Pointers named host_* are host memory, dev_* are device memory.
 *   - calls are asynchronous on `stream` unless the comment says "synchronises".
 *   - objects own their device memory (the 7.06 GB frame ring, weights, activations); getters
 *     expose device pointers for zero-copy interop (torch.as_tensor via __cuda_array_interface__).
 */
#ifndef B200DQN_H
#define B200DQN_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200DQN_VERSION 100 /* 0.1.0 */

enum {
  B200DQN_OK = 0,
  B200DQN_EINVAL = -1,   /* bad argument (the reference would raise AssertionError) */
  B200DQN_ECUDA = -2,    /* CUDA runtime/driver failure, text in b200dqn_last_error() */
  B200DQN_ENOTIMPL = -3, /* a reference flag this build does not implement (NotImplementedError) */
  B200DQN_ENCCL = -4,    /* NCCL failure or libnccl.so.2 not loadable */
  B200DQN_ESTATE = -5    /* call sequence error (e.g. sampling an empty ring) */
};

/* math_mode of b200dqn_net_config */
enum {
  B200DQN_MATH_FP32_SIMT = 0, /* CUDA-core fp32 FFMA implicit GEMM: exact-fp32 reference mode          */
  B200DQN_MATH_TCGEN05 = 1    /* wgmma fp16 hi/lo split operands (3 MMAs), fp32 accumulate    */
};

/* optimizer of b200dqn_net_config — src/deepqnetwork.py:50-61 (--optimizer rmsprop|adam|adadelta, main.py:40) */
enum {
  B200DQN_OPT_RMSPROP = 0,  /* RMSProp(learning_rate, decay_rate), epsilon 1e-6; one state array per W       */
  B200DQN_OPT_ADAM = 1,     /* Adam(learning_rate), beta_1 0.9, beta_2 0.999, epsilon 1e-8; states [m, v]    */
  B200DQN_OPT_ADADELTA = 2  /* Adadelta(decay = decay_rate), epsilon 1e-6; states [E[g^2], E[dx^2], dx]      */
};

typedef struct b200dqn_replay b200dqn_replay; /* replaces class ReplayMemory, src/replay_memory.py:6  */
typedef struct b200dqn_net b200dqn_net;       /* replaces class DeepQNetwork, src/deepqnetwork.py:15 */
typedef struct b200dqn_statebuf b200dqn_statebuf; /* replaces class StateBuffer, src/state_buffer.py:3 */

const char* b200dqn_last_error(void);
int b200dqn_version(void);
/* sm count, compute capability and free/total bytes of `device`; fails unless cc == 10.x */
int b200dqn_device_info(int device, int* sm_count, int* cc_major, int* cc_minor, size_t* free_bytes,
                        size_t* total_bytes);

/* Plain device->host / host->device copies of library-owned memory (tests, checkpointing);
 * both synchronise `stream`. */
int b200dqn_copy_to_host(int device, void* host_dst, const void* dev_src, size_t bytes, void* stream);
int b200dqn_copy_to_device(int device, void* dev_dst, const void* host_src, size_t bytes, void* stream);

/* A non-default (non-blocking) CUDA stream owned by the library, for callers that do not bring their
 * own (torch.cuda.Stream().cuda_stream works too).  The fused train path only uses CUDA-graph
 * replay and side-stream branches when it is given a non-default stream. */
int b200dqn_stream_create(int device, void** out_stream);
int b200dqn_stream_destroy(int device, void* stream);
int b200dqn_stream_synchronize(int device, void* stream);

/* Per-launch timing with CUDA events (bench.py's roofline leg): between begin and end every kernel
 * the library launches is followed by an event on its stream.  end synchronises the device and
 * returns, in launch order, a 32-byte label and the elapsed ms since the previous event. */
int b200dqn_profile_begin(int device, void* stream);
int b200dqn_profile_end(int max_entries, char* names32, float* ms, int* count);

/* In-graph kernel timeline: arm, run ONE fused step (train_fused re-captures its graph with timing
 * slots), then read [label, first CTA start, last CTA end] (GPU %globaltimer, ns) per launch. */
int b200dqn_ktrace_begin(int device);
/* Same, but record only the step-th fused step after arming (step >= 1; run at least that many): a
 * steady-state step out of a batch, which is what a multi-rank trace needs. */
int b200dqn_ktrace_begin_at(int device, int step);
int b200dqn_ktrace_end(int max_entries, char* names32, unsigned long long* start_ns, unsigned long long* end_ns,
                       int* count);

/* ------------------------------------------------------------------ replay ring --------- */

/* ReplayMemory.__init__(size, args)  — src/replay_memory.py:7-24.
 * Allocates screens[size][h][w] u8, actions u8, rewards i64, terminals u8 and the
 * (batch,hist,h,w) prestates/poststates staging in HBM.  batch is the GLOBAL minibatch. */
int b200dqn_replay_create(int device, int64_t size, int screen_h, int screen_w, int history_length,
                          int batch_size, b200dqn_replay** out);
int b200dqn_replay_destroy(b200dqn_replay* r);

/* ReplayMemory.add(action, reward, screen, terminal) — src/replay_memory.py:26-34.
 * host_screen is (h,w) u8; staged through pinned memory, async H2D.  reward is stored as int64
 * (np.integer), so a float reward must be truncated by the caller exactly as numpy does. */
int b200dqn_replay_add(b200dqn_replay* r, int action, int64_t reward, const uint8_t* host_screen,
                       int terminal, void* stream);
/* n consecutive add() calls in one transfer (ring fill / vectorised actors). */
int b200dqn_replay_add_batch(b200dqn_replay* r, int64_t n, const uint8_t* host_actions,
                             const int64_t* host_rewards, const uint8_t* host_screens,
                             const uint8_t* host_terminals, void* stream);
/* the attributes `count` and `current` (src/replay_memory.py:17-18); set is for tests/benches */
int b200dqn_replay_get_cursor(const b200dqn_replay* r, int64_t* count, int64_t* current);
int b200dqn_replay_set_cursor(b200dqn_replay* r, int64_t count, int64_t current);

/* ReplayMemory.getState(index) — src/replay_memory.py:37-48 (negative / wrap-around indexes
 * included).  Writes (hist,h,w) u8 to host_out; synchronises. */
int b200dqn_replay_get_state(b200dqn_replay* r, int64_t index, uint8_t* host_out, void* stream);

/* The random stream of random.randint at src/replay_memory.py:59: CPython's MT19937 state as
 * returned by random.getstate()[1] (624 key words + position).  set uploads it; get downloads
 * the advanced state (synchronises) so the host can random.setstate() and stay in lock-step. */
int b200dqn_replay_set_rng(b200dqn_replay* r, const uint32_t host_mt625[625], void* stream);
int b200dqn_replay_get_rng(b200dqn_replay* r, uint32_t host_mt625[625], void* stream);
/* set_rng without the stream synchronisation, key words and position passed separately (they are separate fields of
 * CPython's generator object): staged through a small pinned ring, asynchronous. */
int b200dqn_replay_set_rng_parts(b200dqn_replay* r, const uint32_t* host_key624, uint32_t host_pos, void* stream);

/* The sampling loop of ReplayMemory.getMinibatch — src/replay_memory.py:55-69 — on the device:
 * draws py3 randint(hist, count-1) trials from the MT19937 stream, applies the two rejection
 * tests (:61, :65) and keeps the first `batch` accepted indexes in acceptance order.
 * Results stay on the device (B200DQN_PTR_INDEXES, B200DQN_PTR_WORDS_CONSUMED). */
int b200dqn_replay_sample(b200dqn_replay* r, void* stream);
/* Same, and returns how many MT19937 words the draw consumed (waits for the sampler only, by polling a host-mapped
 * word — no memcpy, no stream synchronisation): the host keeps its own
 * `random` in lock-step by discarding that many 32-bit words instead of downloading the 2.5 KB state. */
int b200dqn_replay_sample_sync(b200dqn_replay* r, uint32_t* host_words_consumed, void* stream);
/* Test hook: bypass the sampler and use caller-chosen indexes (host int32[batch]). */
int b200dqn_replay_set_indexes(b200dqn_replay* r, const int32_t* host_indexes, void* stream);

/* The copy half of getMinibatch — src/replay_memory.py:71-78: materialises prestates,
 * poststates, actions, rewards, terminals for the sampled indexes in the device staging
 * buffers (TMA bulk copies, one CTA per sample-frame). */
int b200dqn_replay_gather(b200dqn_replay* r, void* stream);

/* Copy the staged minibatch (any pointer may be NULL) to host arrays shaped as the reference
 * returns them: pre/post (batch,hist,h,w) u8, actions u8[batch], rewards i64[batch],
 * terminals u8[batch] (0/1), indexes i32[batch], words_consumed u32[1].  Synchronises. */
int b200dqn_replay_read_minibatch(b200dqn_replay* r, uint8_t* host_pre, uint8_t* host_actions,
                                  int64_t* host_rewards, uint8_t* host_post, uint8_t* host_terminals,
                                  int32_t* host_indexes, uint32_t* host_words_consumed, void* stream);

enum {
  B200DQN_PTR_SCREENS = 0, B200DQN_PTR_ACTIONS, B200DQN_PTR_REWARDS, B200DQN_PTR_TERMINALS,
  B200DQN_PTR_PRESTATES, B200DQN_PTR_POSTSTATES, B200DQN_PTR_MB_ACTIONS, B200DQN_PTR_MB_REWARDS,
  B200DQN_PTR_MB_TERMINALS, B200DQN_PTR_INDEXES, B200DQN_PTR_WORDS_CONSUMED, B200DQN_PTR_MT_STATE,
  /* Prioritized replay (b200dqn_replay_set_prioritized); NULL with 0 bytes until it is first switched on.
   * PRIORITIES: f64[size], the stored priority p^alpha of every slot.  SUM_TREE: f64, the 32-ary sum tree level by
   * level from the leaves (level l has n_l = ceil(n_{l-1} / 32) nodes, n_0 = size, and starts at a multiple of 32
   * entries; the padding is 0).  Leaf i is PRIORITIES[i] if getMinibatch would accept slot i, else 0.  IS_WEIGHTS:
   * f32[batch] of the last draw or set_indexes.  MAX_PRIORITY: f64[1] (not raised to alpha).  MIN_TREE: f64, levels
   * 1.. of the min tree in the same layout (a leaf's min value is itself if positive, else +inf). */
  B200DQN_PTR_PRIORITIES, B200DQN_PTR_SUM_TREE, B200DQN_PTR_IS_WEIGHTS, B200DQN_PTR_MAX_PRIORITY, B200DQN_PTR_MIN_TREE
};
int b200dqn_replay_device_ptr(b200dqn_replay* r, int which, void** dev_ptr, size_t* bytes);

/* Proportional prioritized experience replay (Schaul et al., 2016; the variant of OpenAI baselines'
 * PrioritizedReplayBuffer; new capability, no reference counterpart), off by default.  While it is on:
 *   - the index draw (b200dqn_replay_sample, the fused step) is stratified over the sum tree: sample i takes
 *     mass = random.random() * (total / batch) + i * (total / batch) and descends to the leaf holding it, so a draw
 *     consumes exactly 2 * batch MT19937 words and never draws a slot getMinibatch would reject;
 *   - importance weights w_i = (N P_i)^-beta / (N P_min)^-beta, N = count, beta = beta0 + (1 - beta0) *
 *     min(1, k / beta_steps), k = samplings done, scale each sample's clipped delta and its cost in the train step;
 *   - after a train step on the ring, each sampled slot gets (|delta_i| + eps)^alpha, delta_i the TD error before the
 *     clip (the last occurrence wins for a repeated slot), and max_priority = max(max_priority, |delta_i| + eps);
 *   - slots written by add / add_batch / step_host get max_priority^alpha.
 * Switching on sets every stored priority and max_priority to 1 and builds the trees from the ring as it stands
 * (the first switch-on allocates them).  Either switch rebuilds the captured step graphs of the nets that train from
 * r.  A draw from a ring with no drawable slot reports ESTATE at the next result poll.  Train steps from a
 * prioritized ring return ENOTIMPL for data-parallel learners.  Synchronises. */
int b200dqn_replay_set_prioritized(b200dqn_replay* r, int on, double alpha, double beta0, double beta_steps,
                                   double eps);

/* n-step returns (Hessel et al., 2018; new capability, no reference counterpart), N = n_step, default 1.  With N > 1:
 *   - the draw is randint(hist, count - N) (one MT19937 word per trial, as at N = 1) and rejects a sample whose
 *     window [index - hist, index + N - 1] holds the write pointer (index + N - 1 >= current and index - hist <
 *     current) or whose terminals[index - hist .. index - 1] has a set flag; it needs count >= hist + N;
 *   - the poststate is getState(index + N - 1); b200dqn_replay_gather / read_minibatch stage rewards and terminals
 *     of index .. index + N - 1 as (batch, N) arrays (B200DQN_PTR_MB_REWARDS / _MB_TERMINALS grow to match);
 *   - a train step on the ring forms y = R if a terminal lies in index .. index + N - 1, else R + gamma^N Q^(post),
 *     R = sum_{k<m} gamma^k clip(rewards[index + k]), m the first terminal (or N), in fp64 without contraction;
 *   - the prioritized sum tree masks the same slots.
 * Host-supplied minibatches (b200dqn_net_train / _train_device) stay one-step.  Train steps from a ring with N > 1
 * return ENOTIMPL for data-parallel learners; so does b200dqn_net_comm_init on a net whose last train step used such
 * a ring.  Switching rebuilds the captured step graphs
 * of the nets that train from r.  EINVAL unless 1 <= n and hist + n <= size.  Synchronises. */
int b200dqn_replay_set_n_step(b200dqn_replay* r, int n);

/* ------------------------------------------------------------------ state window -------- */

/* StateBuffer(args) — src/state_buffer.py:9-13: (batch,hist,h,w) u8 zeros on the device. */
int b200dqn_statebuf_create(int device, int screen_h, int screen_w, int history_length, int batch_size,
                            b200dqn_statebuf** out);
int b200dqn_statebuf_destroy(b200dqn_statebuf* s);
/* StateBuffer.add(observation) — src/state_buffer.py:15-18: row 0 shifts left, newest appended. */
int b200dqn_statebuf_add(b200dqn_statebuf* s, const uint8_t* host_screen, void* stream);
/* StateBuffer.reset() — src/state_buffer.py:26-27 */
int b200dqn_statebuf_reset(b200dqn_statebuf* s, void* stream);
/* StateBuffer.getStateMinibatch() / getState() — src/state_buffer.py:20-24; host_out is
 * (batch,hist,h,w) u8 when whole != 0 else (hist,h,w).  Synchronises. */
int b200dqn_statebuf_read(b200dqn_statebuf* s, uint8_t* host_out, int whole, void* stream);
int b200dqn_statebuf_device_ptr(b200dqn_statebuf* s, void** dev_ptr, size_t* bytes);

/* ------------------------------------------------------------------ Q-network ----------- */

typedef struct b200dqn_net_config {
  int num_actions;       /* DeepQNetwork(num_actions, args)        deepqnetwork.py:16-18 */
  int batch_size;        /* args.batch_size (per-rank minibatch)   :19                   */
  int history_length;    /* args.history_length                    :21; 1..16 frames, the
                          * input channels of conv1 (< 1: EINVAL, > 16: ENOTIMPL)        */
  int screen_h, screen_w;/* args.screen_height / width             :22                   */
  double discount_rate;  /* :20  (a Python float: the TD target is formed in double, :141-143) */
  double learning_rate;  /* :51  RMSProp                                                  */
  double decay_rate;     /* :52                                                           */
  double clip_error;     /* :23  (0 disables the clip, as `if self.clip_error:` does)     */
  double min_reward;     /* :24  main.py:43-44 declare both bounds type=float; the reward is clipped  */
  double max_reward;     /* :25  as np.clip(r, min, max) clips: min(max(r, min), max), so max wins if  */
                         /*      the bounds cross                                                     */
  int target_steps;      /* :65  0 ⇒ the target network aliases the online network (:72-73) */
  int math_mode;         /* B200DQN_MATH_*                                                */
  int optimizer;         /* B200DQN_OPT_*  (:50-61; args.optimizer, main.py:40)           */
  /* Distributional value head (C51, Bellemare, Dabney and Munos, 2017; new capability, no reference counterpart),
   * off when num_atoms = 0 (the default).  Otherwise 2..64 atoms on the fixed support z_i = v_min + i dz,
   * dz = (v_max - v_min) / (num_atoms - 1) (fp64), with v_min < v_max both finite (EINVAL otherwise):
   *   - fc2 grows to A * num_atoms outputs (Neon shape (A * num_atoms, 512), row a * num_atoms + i);
   *   - p[a] = softmax(logits[a]) (fp32, row maximum subtracted), Q[a] = sum_i float(z_i) p[a][i] in i order: every
   *     Q output (predict, Q rows) carries these expected values;
   *   - the train step projects the target network's distribution at a* (argmax of its Q, or of the online network's
   *     with Double DQN) onto the support in fp64: T_j = clamp(R + g z_j, v_min, v_max), b_j = (T_j - v_min) / dz,
   *     m_i = float(sum_j q_j max(0, 1 - |b_j - i|)), R the clipped (or n-step) return, g = gamma^N (0 at a terminal);
   *   - the cost is the cross-entropy -sum_i m_i log p[a][i] at the taken action (times the importance weight on a
   *     prioritized ring, whose priority update gets the unweighted loss); clip_error is not applied;
   *   - the logit gradient is (p[a][i] - m_i) w at the taken action and 0 elsewhere.
   * b200dqn_net_comm_init returns ENOTIMPL on such a net. */
  int num_atoms;
  double v_min, v_max;
  /* Dueling network (Wang et al., 2016; new capability, no reference counterpart), off when dueling = 0 (the default;
   * values other than 0 and 1 are EINVAL).  With dueling = 1:
   *   - fc1 has 1024 Rectlin units, Neon shape (1024, 3136): rows 0..511 are the advantage stream, rows 512..1023 the
   *     value stream.  fc2 has Neon shape (A + 1, 512): rows 0..A-1 weigh the advantage units into A_a, row A weighs
   *     the value units into V;
   *   - A_a and V are each formed as the scalar head forms Q (fp32 products, the warp's xor butterfly, the 16 warp
   *     sums in warp order), m = (sum_j A_j in j order) / A, Q_a = V + (A_a - m), every operation rounded on its own.
   *     Every Q output (predict, the Q rows, the TD target, the Double DQN choice) carries this Q;
   *   - the TD step (delta, clip, cost, prioritized and n-step targets) is the scalar head's; backward: g = delta / A,
   *     dA_j = (j == a ? delta - g : -g), dV = delta, dZ4 = (sum_j dA_j W5[j][k], j order) on advantage unit k and
   *     delta W5[A][k] on value unit k, under the H4 mask.  The paper's 1/sqrt(2) rescale of the gradient entering the
   *     convolutions is not applied; its gradient-norm clipping (at 10) is the separate opt-in max_grad_norm.
   * Both engines.  ENOTIMPL with num_atoms > 0; b200dqn_net_comm_init returns ENOTIMPL on such a net. */
  int dueling;
  /* Quantile-regression value head (QR-DQN, Dabney, Rowland, Bellemare and Munos, 2018; new capability, no reference
   * counterpart), off when num_quantiles = 0 (the default).  Otherwise N = num_quantiles in 1..200 (other values are
   * EINVAL), and the Huber threshold is kappa = float(clip_error) (1 by default; 0 gives the pure quantile loss; a
   * non-finite clip_error is EINVAL).  EINVAL with num_atoms > 0 (a net has one head), ENOTIMPL with dueling = 1;
   * b200dqn_net_comm_init returns ENOTIMPL on such a net.  Every operation below is fp32 with its own rounding (no
   * contraction) unless marked fp64; a is the taken action, z the slot (0 online on the prestates, 1 target on the
   * poststates, 2 online on the poststates under Double DQN):
   *    1. midpoints: tau_i = (2i + 1) / 2N in fp64; wlo_i = float(tau_i) weighs u >= 0, whi_i = float((2N - 2i - 1) / 2N)
   *       weighs u < 0;
   *    2. fc2: theta[z][b][a N + i] = sum_k H4[z][b][k] W5[k][a N + i], k = 0..511 in order, as the distributional head's
   *       logits (Neon shape (A N, 512), row a N + i);
   *    3. Q[a] = (sum_i theta[a][i] in i order) / float(N).  Every Q output (predict, the Q rows, the TD choice) is this Q;
   *    4. a* = first index of the maximum of slot 1's Q (slot 2's with Double DQN); q'_j = theta[1][b][a* N + j];
   *    5. the return R and g as for the distributional head, in fp64 (g = 0 when the window holds a terminal);
   *       T_j = float(R + g double(q'_j));
   *    6. u_ij = T_j - theta[0][b][a N + i];
   *    7. w_ij = u_ij < 0 ? whi_i : wlo_i;
   *    8. kappa > 0: L = |u| <= kappa ? 0.5 (u u) : kappa (|u| - 0.5 kappa), rho_ij = (w L) / kappa and
   *       c_ij = (w clamp(u, -kappa, kappa)) / kappa; kappa = 0: rho_ij = w |u|, c_ij = u > 0 ? w : (u < 0 ? -w : 0);
   *    9. Loss_i = (sum_j rho_ij in j order) / N, the row loss l = sum_i Loss_i in i order; the row cost is l (times the
   *       importance weight on a prioritized ring, whose priority update gets the unweighted l);
   *   10. dtheta_i = -((sum_j c_ij in j order) / N), times the importance weight on a prioritized ring; 0 for every other
   *       action;
   *   11. dZ4 and its fp16 planes, and fc2's per-row gradient partials, as for the distributional head with the logit
   *       gradient replaced by dtheta;
   *   12. fc2's gradient is summed as for the distributional head, then the configured optimizer applies it. */
  int num_quantiles;
  /* Munchausen DQN target (M-DQN, Vieillard, Pietquin and Geist, 2020; new capability, no reference counterpart), off
   * when munchausen = 0 (the default; values other than 0 and 1 are EINVAL).  With pi = softmax(q / tau) over a Q row
   * of the target network, the scalar head's target becomes
   *   y = R + alpha clamp(tau ln pi(a | s), l0, 0) + g sum_a' pi(a' | s') (q(s', a') - tau ln pi(a' | s')),
   * R the clipped (or n-step) return and g = gamma^N, 0 when the window holds a terminal (the bonus still applies).
   * alpha = munchausen_alpha (finite, >= 0; default 0.9), tau = munchausen_tau (finite, > 0; default 0.03) and
   * l0 = munchausen_clip (finite, <= 0; default -1); anything else is EINVAL.  ENOTIMPL with dueling, num_atoms or
   * num_quantiles; b200dqn_net_set_double_q(n, 1) is EINVAL (the target makes no greedy choice) and
   * b200dqn_net_comm_init returns ENOTIMPL on such a net.  The train step runs the target network on the prestates
   * as one more forward pass (no pass with target_steps = 0: the online Q row of the prestates is that row).  Every
   * fp64 operation below is rounded on its own except exp and log, which are the device's fp64 functions (not
   * bit-identical to numpy's); a is the taken action:
   *    1. per sample, two fp32 rows x: the target network's Q on the poststates, and its Q on the prestates.  For each
   *       row: m = max_j x_j; e_j = exp((double(x_j) - m) / tau); s = sum_j e_j in j order; lse = m + tau log(s);
   *       tau ln pi_j = double(x_j) - lse; pi_j = e_j / s;
   *    2. bonus = alpha fmin(fmax(tau ln pi_pre[a], l0), 0);
   *    3. next = sum_j pi_post,j (x_post,j - tau ln pi_post,j) in j order;
   *    4. y = (R + bonus) + g next, the last operation formed as the scalar head forms its one-step (contracted) and
   *       n-step (separately rounded) targets, so that with one action y is the scalar head's y bit for bit;
   *    5. target = float(y); delta, the clip, the importance weight, the cost, the TD error, dZ4 and fc2's gradient
   *       are the scalar head's. */
  int munchausen;
  double munchausen_alpha;
  double munchausen_tau;
  double munchausen_clip;
  /* Implicit quantile network head (IQN, Dabney, Ostrovski, Silver and Munos, 2018; new capability, no reference
   * counterpart), off when num_tau_samples = 0 (the default).  Otherwise N = num_tau_samples in 1..64 and
   * K = num_quantile_samples in 1..64 (default 32), with nb max(N, K) <= 4096 rows (EINVAL otherwise, before any
   * device work); kappa = float(clip_error) as for the quantile-regression head (non-finite: EINVAL).  EINVAL with
   * num_atoms or num_quantiles (a net has one head), ENOTIMPL with dueling or munchausen;
   * b200dqn_net_set_double_q(n, 1) and b200dqn_net_comm_init return ENOTIMPL on such a net.  The embedding is ABI layer
   * 5, Neon shape (3136, 64) (row n = fc1's input column in Neon's (c, p, q) order), with its own optimizer states; it
   * belongs to each network (online and target) like every other layer.  b is the sample, a the taken action, z the
   * slot (0 online on the prestates, 1 target on the poststates); every fp32 operation is rounded on its own:
   *    1. tau draw: tau = (2m + 1) 2^-24, m = h >> 9 where h is the high 32 bits of
   *         x = mix(mix(tau_seed + 0x9E3779B97F4A7C15 (ctr + 1)) ^ (z << 32 | b << 8 | j)),
   *       mix = splitmix64's finaliser (x ^= x >> 30; x *= 0xBF58476D1CE4E5B9; x ^= x >> 27; x *= 0x94D049BB133111EB;
   *       x ^= x >> 31), all mod 2^64, ctr the device-resident draw counter.  Every forward (train step or predict)
   *       draws with the counter's value and then advances it by one, on the device, so replayed step and predict
   *       graphs draw fresh tau; the replay sampler's MT19937 stream is not touched;
   *    2. rows r = b N + j (train: N online rows on slot 0, N target rows on slot 1), r = b K + k on predict (slot 0);
   *    3. c[r][i] = float(cos((pi i) tau_r)) for i = 0..63, formed in fp64 with the device's cos (c[r][0] = 1 is the
   *       embedding's bias);
   *    4. phi[r][col] = max(0, sum_i c[r][i] We[i][col], i order), We of the slot's network;
   *    5. X[r] = psi[b] * phi[r], psi = conv3's Rectlin output H3 of the sample; fc1 and fc2 run on X at nb N rows
   *       (nb K on predict) with the scalar net's kernels;
   *    6. theta[z][r][a] = sum_k H4[z][r][k] W5[k][a], k = 0..511 in order;
   *    7. Q[a] = (sum_j theta[b N + j][a], j order) / float(N) per slot (K on predict).  Every Q output is this Q;
   *    8. a* = first index of the maximum of slot 1's Q (a simplification: the paper draws K separate samples for a*);
   *    9. T_j = float(R + g double(theta[1][b N + j][a*])), R and g as for the quantile-regression head;
   *       u_ij = T_j - theta[0][b N + i][a], weight tau_i (slot 0's tau of row b N + i) for u >= 0 and 1 - tau_i for
   *       u < 0; the loss, the row cost, the importance weight, the priority and dtheta_i then follow rules 8-10 of
   *       the quantile-regression head over the N x N pairs;
   *   10. dZ4[r][k] = H4[0][r][k] > 0 ? W5[k][a] dtheta_r : 0; fc2's gradient is sum_r H4[0][r][k] dtheta_r in row
   *       order at column a, then the configured optimizer (batch size nb) applies it;
   *   11. dX = fc1's dgrad at nb N rows (masked by X > 0, harmless: X = psi phi >= 0, and where X = 0 both terms of 12
   *       vanish anyway);
   *   12. dpsi[b][col] = (sum_j dX[b N + j][col] phi[b N + j][col], j order), 0 unless psi > 0; it is conv3's dZ (the
   *       DZ3 selector); dphi[r][col] = phi > 0 ? dX[r][col] psi[b][col] : 0;
   *   13. dWe[i][col] = sum_r c[r][i] dphi[r][col] over slot 0's rows in row order; the configured optimizer (batch size
   *       nb) applies it. */
  int num_tau_samples;
  int num_quantile_samples;
  uint64_t tau_seed;
  /* Random-shift augmentation (DrQ, Kostrikov, Yarats and Fergus, 2020; new capability, no reference counterpart), off
   * when random_shift = 0 (the default).  Otherwise p = random_shift in 1..8 (DrQ uses 4; other values are EINVAL,
   * before any device work), and every train step trains on shifted states.  b200dqn_net_comm_init returns ENOTIMPL
   * on such a net.  b is the sample, z the slot (0 the prestates, 1 the poststates):
   *    1. draw: x = mix(mix(shift_seed + 0x9E3779B97F4A7C15 (ctr + 1)) ^ (z << 32 | b)),
   *         dy = ((x >> 32) (2p + 1) >> 32) - p,   dx = ((x & 0xffffffff) (2p + 1) >> 32) - p,
   *       all mod 2^64, mix = the IQN head's splitmix64 finaliser, ctr the device-resident draw counter of the shift
   *       (not the IQN head's).  Every train step, on every train entry point, draws with the counter's value and then
   *       advances it by one, on the device, so replayed step graphs draw fresh offsets; predict, its graph and acting
   *       neither shift nor touch the counter; the replay sampler's MT19937 stream is not touched;
   *    2. the shifted state's pixel (f, y, x) is frame f's pixel (clamp(y + dy, 0, 83), clamp(x + dx, 0, 83)): one
   *       (dy, dx) for all history_length frames of a state; this is edge-replicate padding by p followed by the 84x84
   *       crop at (p + dy, p + dx);
   *    3. the online network on the prestates (slot 0) and the Munchausen target pass on the prestates read slot 0's
   *       offsets; the target network on the poststates (slot 1) and Double DQN's online network on the poststates
   *       read slot 1's.  The stored frames, and what getMinibatch returns, are never shifted. */
  int random_shift;
  uint64_t shift_seed;
  /* Random ensemble mixture head (REM, Agarwal, Schuurmans and Norouzi, 2020; new capability, no reference counterpart),
   * off when num_heads = 0 (the default).  Otherwise K = num_heads in 1..200 (other values are EINVAL) Q-value heads
   * per action, mixed by one random convex combination per train step.  EINVAL with num_atoms, num_quantiles or
   * num_tau_samples (a net has one head), ENOTIMPL with dueling or munchausen; b200dqn_net_comm_init returns ENOTIMPL
   * and the DELTAS selector is EINVAL on such a net.  Every fp32 operation below is rounded on its own (no
   * contraction) unless marked fp64; a is the taken action, z the slot (0 online on the prestates, 1 target on the
   * poststates, 2 online on the poststates under Double DQN):
   *    1. mixture draw, once per train step: u_k = (2 m_k + 1) 2^-24, m_k = h >> 9 where h is the high 32 bits of
   *         x = mix(mix(rem_seed + 0x9E3779B97F4A7C15 (ctr + 1)) ^ k)
   *       (the IQN head's tau hash at z = 0, b = 0, j = k), ctr the mixture's device-resident draw counter;
   *       S = sum_k double(u_k) in fp64, k order; alpha_k = float(double(u_k) / S).  The same alpha serves every sample
   *       and slot of the step.  Every train step, on every train entry point, draws with the counter's value and then
   *       advances it by one, on the device, so replayed step graphs draw fresh alpha; predict neither reads nor
   *       advances it; the replay sampler's MT19937 stream is not touched;
   *    2. fc2: theta[z][b][a K + k] = sum_i H4[z][b][i] W5[i][a K + k], i = 0..511 in order, as the distributional
   *       head's logits (Neon shape (A K, 512), row a K + k);
   *    3. train-step Q: Q[z][a] = sum_k alpha_k theta[z][b][a K + k] in k order (each product rounded, then each sum).
   *       The Q rows of a train step, the greedy target and the Double DQN choice use this Q;
   *    4. predict Q: Q[a] = (sum_k theta[a][k] in k order) / float(K), the quantile-regression head's rule 3;
   *    5. the TD step is the scalar head's on the rule-3 Q: the clipped (or n-step) return, the maximum of slot 1's Q
   *       (slot 1's Q at the first maximum of slot 2's with Double DQN), y = R + g maxq (one fused multiply-add on the
   *       one-step step, a separately rounded product and sum on the n-step step), target = float(y),
   *       delta = Q[0][a] - target; the row cost 0.5 delta delta (times the importance weight w on a prioritized ring,
   *       whose TD error is delta); d = clamp(delta, -clip_error, clip_error) (no clip when clip_error = 0), times w on
   *       a prioritized ring;
   *    6. dtheta[a][k] = alpha_k d at the taken action, 0 for every other action;
   *    7. dZ4 and its fp16 planes, and fc2's per-row gradient partials, as for the distributional head with the logit
   *       gradient replaced by dtheta; fc2's gradient is summed as for the distributional head (block width K), then
   *       the configured optimizer applies it. */
  int num_heads;
  uint64_t rem_seed;
  /* Fully parameterized quantile function head (FQF, Yang, Zhao, Lin, Qin, Bian and Liu, 2019; new capability, no
   * reference counterpart), off when num_fractions = 0 (the default).  Otherwise N = num_fractions in 2..64 with
   * nb N <= 4096 rows, and fraction_lr (finite, >= 0) is the learning rate of the fraction proposal layer; anything else
   * is EINVAL before any device work, as are num_atoms, num_quantiles, num_tau_samples or num_heads beside it (a net has
   * one head) and a non-finite clip_error.  ENOTIMPL with dueling or munchausen; b200dqn_net_set_double_q(n, 1) and
   * b200dqn_net_comm_init return ENOTIMPL on such a net.  ABI layer 5 is the IQN head's embedding (Neon shape
   * (3136, 64)), ABI layer 6 the fraction layer W_f (Neon shape (N, 3136), columns in fc1's Neon (c, p, q) input order);
   * both have optimizer states and belong to each network, and the step reads the online W_f only.  kappa, b, a, z and
   * the rounding are as for the IQN head; psi is the online network's fp32 H3 of the prestates; every fp64 operation
   * is rounded on its own except exp, the device's fp64 exp:
   *    1. logits l[b][k] = sum over col of psi[b][col] W_f[k][col] in fc1's internal (p, q, c) column order, as 32
   *       lanes: lane j sums the products of columns j, j + 32, ..., j + 3104 in order, then the lanes are combined by
   *       halving, s_j = s_j + s_{j + h} for h = 16, 8, 4, 2, 1;
   *    2. proposal in fp64: m = max_k l_k; e_k = exp(double(l_k) - m); C_0 = 0, C_{i+1} = C_i + e_i in i order,
   *       S = C_N; q_k = float(e_k / S); tau_i = float(C_i / S) (tau_0 = 0, tau_N = 1); tauhat_i =
   *       float((C_i + C_{i+1}) / (2 S)).  With zero logits tauhat is the quantile-regression head's midpoints;
   *    3. rows r = b N + i: slot 0 the online network at tauhat on the prestates, slot 1 the target network at the
   *       same tauhat on the poststates; each slot runs the IQN head's rules 3-6 (c, phi, X = psi phi, fc1, fc2);
   *    4. Q[a] = sum_i dtau_i theta[b N + i][a] in i order (each product rounded, then each sum), dtau_i =
   *       tau_{i+1} - tau_i.  Every Q output is this Q: predict, the Q rows, and a* = the first maximum of slot 1's Q
   *       (a simplification: the target is valued at the prestates' proposal, not at a second proposal on the
   *       poststates);
   *    5. the quantile loss, the row cost, the importance weight, the priority (the unweighted row loss), dtheta, dZ4
   *       and its planes, fc2's gradient, dpsi, dphi and dWe are the IQN head's rules 9-13 with weight tauhat_i; tauhat
   *       is a constant to this loss and W_f gets no gradient from it;
   *    6. boundary pass, forward only, on the online network at tau_1..tau_{N-1}: rows b (N - 1) + i - 1 through the
   *       IQN head's rules 3-6 give theta_bnd; beta_i = theta_bnd[b (N - 1) + i - 1][a];
   *    7. fraction gradient, i = 1..N-1: g_i = (2 beta_i - theta[0][b N + i][a]) - theta[0][b N + i - 1][a], times
   *       the importance weight on a prioritized ring; dq_k = sum_{i = k+1..N-1} g_i accumulated from i = N - 1
   *       downward (dq_{N-1} = 0); s = sum_k q_k dq_k in k order; dl_k = q_k (dq_k - s);
   *    8. dW_f[k][col] = sum_b dl[b][k] psi[b][col] in b order; the configured optimizer (batch size nb, its other
   *       hyperparameters and Adam's t the net's) applies it with learning rate fraction_lr.  psi gets no gradient
   *       from the fraction loss. */
  int num_fractions;
  double fraction_lr;
  /* Bootstrapped DQN heads (Osband, Blundell, Pritzel and Van Roy, 2016; new capability, no reference counterpart), off
   * when bootstrap_heads = 0 (the default).  Otherwise K = bootstrap_heads in 1..200 Q-value heads per action on the
   * shared network, each trained on its own target and masked by its own bootstrap mask, with mask probability p =
   * bootstrap_p, finite, in (0, 1].  A bad K or p is EINVAL before any device work, as are num_atoms, num_quantiles,
   * num_tau_samples, num_heads or num_fractions beside it (a net has one head); ENOTIMPL with dueling or munchausen.
   * b200dqn_net_comm_init returns ENOTIMPL on such a net, and the DELTAS, REM_ALPHAS and REM_COUNTER selectors are
   * EINVAL; REM_HEADS and REM_GRADS read theta and dtheta.  With p < 1, b200dqn_net_train and b200dqn_net_train_device
   * return ENOTIMPL (their rows are no ring slots, so they carry no mask); at p = 1 they train.  Every fp32 operation
   * below is rounded on its own (no contraction) unless marked fp64; b is the sample, a the taken action, z the slot
   * (0 online on the prestates, 1 target on the poststates, 2 online on the poststates under Double DQN), i the ring
   * slot the step reads the sample's transition from:
   *    1. masks: m_k(b) = [double(u) < p] with u = (2 (h >> 9) + 1) 2^-24, h the high 32 bits of
   *         x = mix(mix(bootstrap_seed + 0x9E3779B97F4A7C15 (i + 1)) ^ k)
   *       (the REM head's draw at counter i).  The mask belongs to the ring slot: every step that draws slot i, on any
   *       entry point, in any graph replay, sees the same mask; at p = 1 every mask is 1;
   *    2. fc2: theta[z][b][a K + k] as the REM head's rule 2 (Neon shape (A K, 512));
   *    3. per-head targets: a*_k = the first maximum over a of slot 1's theta[a K + k] (slot 2's with Double DQN);
   *       y_k = R + g theta[1][b][a*_k K + k] (one fused multiply-add on the one-step step, a separately rounded
   *       product and sum on the n-step step, R at a terminal) with the scalar head's clipped (or n-step) return R and
   *       g, target_k = float(y_k), delta_k = theta[0][b][a K + k] - target_k;
   *    4. loss: row cost = (sum_k m_k 0.5 delta_k delta_k in k order) / float(K), times the importance weight w on a
   *       prioritized ring, whose TD error is (sum_k |delta_k| in k order) / float(K) over every head, masked or not;
   *       d_k = clamp(delta_k, -clip_error, clip_error) (no clip when clip_error = 0), times w on a prioritized ring;
   *       dtheta[a][k] = m_k ? d_k : 0 at the taken action, 0 for every other action;
   *    5. backward: dZ4[t] = H4[t] > 0 ? (sum_k W5[t][a K + k] dtheta_k in k order) / float(K) : 0 (the gradient
   *       entering the shared network is the mean over the heads), with the fp16 planes every head writes; fc2's
   *       per-row partials are H4[t] dtheta_k, summed as for the REM head (block width K), then the configured
   *       optimizer applies them;
   *    6. the Q rows of a train step are rule 7's at h = -1 (nothing in the step reads them);
   *    7. predict at the active head h (a device-resident int32, -1 after creation): h = -1 gives Q[a] = (sum_k
   *       theta[a][k] in k order) / float(K), the REM head's predict Q; h >= 0 gives Q[a] = theta[a][h].  A predict
   *       enqueued after b200dqn_net_set_active_head sees its h, on every predict entry point, including a replay
   *       of the captured fast-path graph, which is not recaptured. */
  int bootstrap_heads;
  double bootstrap_p;
  uint64_t bootstrap_seed;
  /* Soft (Polyak-averaged) target-network update (new capability, no reference counterpart; SB3's and CleanRL's `tau`),
   * off when soft_target_tau = 0 (the default).  Otherwise tau = soft_target_tau, finite, in (0, 1] (anything else is
   * EINVAL, as is tau > 0 with target_steps = 0: there is no separate target to blend; both before any device work),
   * and every train step, on every train entry point, ends by blending each layer of the target network towards the
   * online one.  b200dqn_net_comm_init returns ENOTIMPL on such a net.  Both engines.  Per element, every operation
   * rounded on its own (no contraction):
   *    1. c = float(1 - tau), 1 - tau formed in fp64 from the config double; t = float(tau);
   *    2. theta_target' = fl(fl(c theta_target) + fl(t theta)), theta the online weight after this step's optimizer
   *       update;
   *    3. it covers layers 0-4, the IQN / FQF embedding (layer 5) and the FQF fraction layer (layer 6); the target's
   *       optimizer state planes are not touched (only b200dqn_net_sync_target copies them);
   *    4. on the tensor-core engine the target's forward tile images after the step are the packing of the new fp32
   *       target weights, the images b200dqn_net_set_weights(which = 1) builds.
   * At tau = 1 the target equals the online weights in value (c = 0, t = 1; an online -0 may land as +0).  The hard
   * copy b200dqn_net_sync_target keeps working beside it. */
  double soft_target_tau;
  /* Global gradient-norm clipping (new capability, no reference counterpart; SB3's `max_grad_norm`, OpenAI baselines'
   * `grad_norm_clipping`, the dueling paper's clip at 10), off when max_grad_norm = 0 (the default): the step is then
   * exactly the unclipped step.  A negative, NaN or infinite value is EINVAL before any device work.
   * b200dqn_net_comm_init returns ENOTIMPL on such a net.  Both engines, every head, every train entry point (train,
   * train_device, train_fused, step_host, replayed graphs), both schedules.  With M = max_grad_norm > 0 each train step:
   *    1. for every parameter of layers 0-4 and of the IQN / FQF embedding (layer 5) forms gg = fl32(g / bsz), exactly
   *       the value the unclipped update forms: g is the summed gradient the unclipped update reads (what
   *       b200dqn_net_get_grads returns), bsz the optimizer's batch size (nb on every layer, the expanded IQN / FQF
   *       layers included);
   *    2. S_l = sum of double(gg)^2 over layer l in fp64 (the products are exact), in an order fixed by the
   *       implementation (no floating-point atomics: two runs give the same bits); S_5 = 0 without an embedding;
   *    3. N = sqrt(S_0 + S_1 + ... + S_5) in fp64, summed in layer order;
   *    4. c = M / (N + 1e-6) in fp64, c32 = (c < 1.0) ? float(c) : 1.0f (torch's clip_grad_norm_ coefficient; a NaN N
   *       gives c32 = 1, so NaN gradients pass through as they do unclipped; an infinite N gives c32 = 0);
   *    5. gg' = fl32(gg c32), and the configured optimizer continues from gg' in its usual operation order (Adam's step
   *       scalar is unchanged).  At c32 = 1, gg' = gg: a net whose norm never reaches M trains bit for bit like a net
   *       without clipping;
   *    6. the FQF fraction layer (layer 6) is neither counted nor scaled: it has its own learning rate (in the FQF
   *       paper its own optimizer) and updates exactly as unclipped.
   * b200dqn_net_get_grads keeps returning the pre-clip g; soft target blends follow the clipped update.  The GRAD_SQ,
   * GRAD_NORM and CLIP_SCALE selectors read S_l, N and c32 of the last train step.  This follows torch and SB3, not
   * Neon: Neon's gradient_clip_norm scales only the step and divides the norm by the batch size, and its
   * gradient_clip_value clips each element; neither is what the configurations this field ports mean. */
  double max_grad_norm;
} b200dqn_net_config;

int b200dqn_net_config_default(b200dqn_net_config* cfg, int num_actions);

/* DeepQNetwork.__init__ — src/deepqnetwork.py:16-75.  Weights start at zero: the caller
 * initialises them with b200dqn_net_set_weights (Xavier draw or a snapshot). */
int b200dqn_net_create(int device, const b200dqn_net_config* cfg, b200dqn_net** out);
int b200dqn_net_destroy(b200dqn_net* n);

/* Weights cross the boundary in NEON layout: conv W[C*R*S][K], linear W[nout][nin], fp32,
 * C-contiguous (what Model.get_description / the shipped snapshots hold); host_S is the
 * RMSProp state of the same shape (may be NULL).  layer 0..4 (and 5, the embedding, on an IQN or FQF net; 6, the fraction
 * layer, on an FQF net); which 0 = online,
 * 1 = target.
 * Replaces Model.load_params / save_params — src/deepqnetwork.py:188-192.  Synchronises. */
int b200dqn_net_set_weights(b200dqn_net* n, int which, int layer, const float* host_W, const float* host_S,
                            void* stream);
int b200dqn_net_get_weights(b200dqn_net* n, int which, int layer, float* host_W, float* host_S, void* stream);
int b200dqn_net_layer_shape(const b200dqn_net* n, int layer, int* rows, int* cols);
/* Optimizer state plane k of `layer` (Neon's `states[k]`: RMSProp k = 0; Adam k = 0 m, 1 v; Adadelta k = 0..2),
 * NEON layout like the weights.  b200dqn_net_num_states returns how many planes the configured optimizer keeps.
 * Both synchronise. */
int b200dqn_net_num_states(const b200dqn_net* n, int* count);
int b200dqn_net_set_state(b200dqn_net* n, int which, int layer, int k, const float* host_S, void* stream);
int b200dqn_net_get_state(b200dqn_net* n, int which, int layer, int k, float* host_S, void* stream);

/* DeepQNetwork.update_target_network — src/deepqnetwork.py:102-105 (weights and optimizer state). */
int b200dqn_net_sync_target(b200dqn_net* n, void* stream);
/* One soft target update at tau outside a train step, by the rule of b200dqn_net_config::soft_target_tau and its
 * kernels (with tau in place of soft_target_tau): the interval form, a blend every k-th train step.  Any net with a
 * separate target network, whatever its soft_target_tau.  EINVAL unless tau is finite in (0, 1], and with
 * target_steps = 0.  Asynchronous, in stream order. */
int b200dqn_net_soft_update_target(b200dqn_net* n, double tau, void* stream);

/* DeepQNetwork.predict(states) — src/deepqnetwork.py:174-186.  host_states (batch,hist,h,w) u8,
 * host_q (batch,A) f32 (already transposed as `qvalues.T`).  H2D + forward + D2H; synchronises. */
int b200dqn_net_predict(b200dqn_net* n, const uint8_t* host_states, float* host_q, void* stream);
/* Same on device memory; rows >= live_rows must be all-zero frames (the StateBuffer case,
 * agent.py:55-58): they are padding, not computed, and dev_q rows >= live_rows are written as
 * exact zeros (not the network's value there, which a distributional head makes mean(z)).
 * live_rows = batch computes everything.  Asynchronous. */
int b200dqn_net_predict_device(b200dqn_net* n, const uint8_t* dev_states, int live_rows, float* dev_q,
                               void* stream);

/* The agent's action selection (src/agent.py:55-61) on a device-resident state window: forward for the live rows as ONE
 * captured CUDA graph, Q-values back through host-mapped memory (no memcpy; the call polls).  host_q is (batch, A);
 * rows >= live_rows are exact zeros.  Needs a non-default stream for the graph path (falls back to
 * b200dqn_net_predict_device + copy otherwise).  Synchronises on the result only. */
int b200dqn_net_predict_device_host(b200dqn_net* n, const uint8_t* dev_states, int live_rows, float* host_q,
                                    void* stream);

/* DeepQNetwork.train(minibatch, epoch) — src/deepqnetwork.py:107-172 — from HOST arrays as the
 * reference passes them (drop-in mode).  terminals is u8 0/1.  host_cost receives cost[0,0]
 * (:171); synchronises. */
int b200dqn_net_train(b200dqn_net* n, const uint8_t* host_pre, const uint8_t* host_actions,
                      const int64_t* host_rewards, const uint8_t* host_post, const uint8_t* host_terminals,
                      float* host_cost, void* stream);
/* Same from device-resident minibatch buffers (what b200dqn_replay_gather produced). Async. */
int b200dqn_net_train_device(b200dqn_net* n, const uint8_t* dev_pre, const uint8_t* dev_actions,
                             const int64_t* dev_rewards, const uint8_t* dev_post, const uint8_t* dev_terminals,
                             void* stream);
/* agent.py:112-114 fused: `nsteps` × (getMinibatch sampling → frames read straight from the ring
 * by the first conv layer → train).  No staging copy, no host round trip.  In a multi-GPU
 * communicator every rank samples the same global minibatch and trains on its own slice.
 * Asynchronous; costs land in the device cost ring (b200dqn_net_read_costs). */
int b200dqn_net_train_fused(b200dqn_net* n, b200dqn_replay* r, int nsteps, void* stream);
/* One train step on the indexes ALREADY sampled into the replay object (b200dqn_replay_sample /
 * _set_indexes): the `net.train(mem.getMinibatch())` pair of agent.py:112-114 when getMinibatch
 * returned a device handle.  Frames are read in place from the ring.  Asynchronous. */
int b200dqn_net_train_sampled(b200dqn_net* n, b200dqn_replay* r, void* stream);
/* Same, then returns cost[0,0] of this step in host_cost (written to host-mapped memory by the step's cost kernel; the
 * call polls that word: no memcpy, no stream synchronisation — the rest of the step may still be running) for the
 * `callback.on_train(cost)` of src/deepqnetwork.py:171-172. */
int b200dqn_net_train_sampled_cost(b200dqn_net* n, b200dqn_replay* r, float* host_cost, void* stream);
/* src/agent.py:102-114 as ONE call, for a caller that drives the loop itself (one host->device hop per train step):
 *   nframes x ReplayMemory.add (the env steps since the last train; frames are (h,w) u8, back to back), then
 *   train_repeat x (ReplayMemory.getMinibatch sampling + DeepQNetwork.train) as captured CUDA graphs.
 * host_key624 != NULL: the caller drew from its `random` since the last call — the MT19937 state (624 key words,
 * position) is adopted first.  host_costs (train_repeat floats) / host_words_consumed (MT words the samplings
 * consumed, so the caller can advance its `random`) arrive through host-mapped memory written by the kernels: no
 * memcpy, one wait.  Both NULL: the call is asynchronous.  train_repeat = 0 only appends the frames. */
int b200dqn_net_step_host(b200dqn_net* n, b200dqn_replay* r, int nframes, const uint8_t* host_actions,
                          const int64_t* host_rewards, const uint8_t* host_frames, const uint8_t* host_terminals,
                          int train_repeat, const uint32_t* host_key624, uint32_t host_pos, float* host_costs,
                          uint32_t* host_words_consumed, void* stream);
/* The last `count` (<= 1024) per-step costs, oldest first.  Synchronises. */
int b200dqn_net_read_costs(b200dqn_net* n, int count, float* host_costs, void* stream);
/* train_iterations — src/deepqnetwork.py:168 */
int b200dqn_net_train_iterations(const b200dqn_net* n, int64_t* iters);

enum {
  B200DQN_NET_PTR_Q_ONLINE = 0, /* preq  (batch,A) f32 of the last train/predict — deepqnetwork.py:129 */
  B200DQN_NET_PTR_Q_TARGET,     /* postq (batch,A) f32 — :120                                          */
  B200DQN_NET_PTR_DELTAS,       /* clipped deltas (batch,A) f32 — :159                                 */
  B200DQN_NET_PTR_GRADS,        /* summed dW, internal layout, all layers contiguous                   */
  B200DQN_NET_PTR_WEIGHTS,      /* online fp32 master weights, internal layout                         */
  B200DQN_NET_PTR_COST,         /* device cost ring                                                    */
  B200DQN_NET_PTR_H1,           /* online activations of the last forward, NHWC fp32: (batch,20,20,32) */
  B200DQN_NET_PTR_H2,           /* (batch,9,9,64)                                                      */
  B200DQN_NET_PTR_H3,           /* (batch,7,7,64)                                                      */
  B200DQN_NET_PTR_H4,           /* (batch,512); (batch,1024) on a dueling net                           */
  /* Online-network gradients at each layer's pre-activation (Rectlin mask applied) of the last train step, NHWC
   * fp32.  DZ4 is always written.  DZ3..DZ1 are always written by the FP32_SIMT engine; the tensor-core engine writes
   * them only while b200dqn_net_set_keep_grads is on, otherwise they hold whatever was there before. */
  B200DQN_NET_PTR_DZ4,          /* (batch,512); (batch,1024) on a dueling net                           */
  B200DQN_NET_PTR_DZ3,          /* (batch,7,7,64)                                                      */
  B200DQN_NET_PTR_DZ2,          /* (batch,9,9,64)                                                      */
  B200DQN_NET_PTR_DZ1,          /* (batch,20,20,32)                                                    */
  /* The online network's Q on the poststates of the last Double DQN train step, (batch,A) f32: the row whose first
   * maximum picks the action the target network values.  With target_steps = 0 it is the Q_TARGET buffer (the two
   * networks are one). */
  B200DQN_NET_PTR_Q_ONLINE_POST,
  /* (batch,) f32: the TD error delta_i = preq[a_i] - target_i before the clip, of the last train step on a
   * prioritized ring (the quantity its priority update uses).  EINVAL before the first such step. */
  B200DQN_NET_PTR_TD_ERRORS,
  /* (batch,) f32: the per-sample cost 0.5*delta^2 before the clip (times the importance weight on a prioritized ring)
   * of the last train step, whose mean in row order is the step's cost.  Distributional head: the cross-entropy. */
  B200DQN_NET_PTR_ROW_COSTS,
  /* Distributional head only (num_atoms > 0; EINVAL otherwise).  DELTAS is EINVAL on such a net: there is no scalar
   * delta.  Slots as in the forward: 0 online on the prestates, 1 target on the poststates, 2 online on the
   * poststates (Double DQN). */
  B200DQN_NET_PTR_LOGITS,       /* (3, batch, A * num_atoms) f32 fc2 outputs of the last forward         */
  B200DQN_NET_PTR_PROBS,        /* (3, batch, A, num_atoms) f32 softmax of each action's logits           */
  B200DQN_NET_PTR_TARGET_DIST,  /* (batch, num_atoms) f32 projected target distribution m                 */
  B200DQN_NET_PTR_LOGIT_GRADS,  /* (batch, num_atoms) f32 gradient on the taken action's logits           */
  /* Tensor-core engine only (EINVAL on the SIMT engine): the fp16 planes of DZ4 the tensor-core dgrad reads, hi then
   * lo (scaled by 2048), each (batch, 512) row-major, (batch, 1024) on a dueling net; the lo plane starts
   * bytes / 2 - batch * width elements after hi. */
  B200DQN_NET_PTR_DZ4_PLANES,
  /* Dueling net only (EINVAL otherwise): (3, batch, A + 1) f32, the advantages A_0..A_{A-1} and then V of each row of
   * the last forward, slots as for the distributional head (slot 2 is written by Double DQN steps with a separate
   * target network only). */
  B200DQN_NET_PTR_DUELING_VA,
  /* Quantile-regression head only (num_quantiles > 0; EINVAL otherwise).  DELTAS is EINVAL on such a net.  Slots as for
   * the distributional head. */
  B200DQN_NET_PTR_QUANTILES,        /* (3, batch, A * num_quantiles) f32 fc2 outputs theta of the last forward      */
  B200DQN_NET_PTR_TARGET_QUANTILES, /* (batch, num_quantiles) f32 target quantiles T_j of the last train step       */
  B200DQN_NET_PTR_QUANTILE_GRADS,   /* (batch, num_quantiles) f32 gradient dtheta on the taken action's quantiles   */
  /* Munchausen target only (munchausen = 1; EINVAL otherwise). */
  B200DQN_NET_PTR_Q_TARGET_PRE,     /* (batch, A) f32 the target network's Q on the prestates of the last train step;
                                     * with target_steps = 0 it is the Q_ONLINE buffer (the two networks are one)   */
  B200DQN_NET_PTR_TD_TARGETS,       /* (batch,) f32 the targets float(y) of the last train step                     */
  /* IQN head only (num_tau_samples > 0; EINVAL otherwise).  Rows as in its rules: nb N per slot after a train step, nb K
   * on slot 0 after a predict; R = nb max(N, K) rows are reserved per slot.  H4 and DZ4 hold R rows on such a net, DZ3
   * is dpsi, and the quantile-regression selectors and DELTAS are EINVAL. */
  B200DQN_NET_PTR_IQN_TAUS,         /* (2, R) f32 tau of the last forward                                            */
  B200DQN_NET_PTR_IQN_COS,          /* (2, R, 64) f32 cosine features c                                              */
  B200DQN_NET_PTR_IQN_PHI,          /* (2, R, 3136) f32 embedding output phi, fc1's internal (p, q, c) column order  */
  B200DQN_NET_PTR_IQN_X,            /* (2, R, 3136) f32 fc1's input X = psi * phi, same order                        */
  B200DQN_NET_PTR_IQN_QUANTILES,    /* (2, R, A) f32 theta                                                           */
  B200DQN_NET_PTR_IQN_TARGET_QUANTILES, /* (batch, N) f32 T_j of the last train step                                 */
  B200DQN_NET_PTR_IQN_QUANTILE_GRADS,   /* (batch N,) f32 dtheta of the taken action, per online row                 */
  B200DQN_NET_PTR_IQN_DX,           /* (R, 3136) f32 fc1's dgrad dX of the last train step                           */
  B200DQN_NET_PTR_IQN_DPHI,         /* (R, 3136) f32 dphi of the last train step                                     */
  B200DQN_NET_PTR_IQN_TAU_COUNTER,  /* u64 the draw counter (the next forward draws with this value)                 */
  /* Random-shift augmentation only (random_shift > 0; EINVAL otherwise). */
  B200DQN_NET_PTR_SHIFT_OFFSETS,    /* (2, batch, 2) i32 (dy, dx) of the last train step: prestates, then poststates */
  B200DQN_NET_PTR_SHIFT_DRAWS,      /* u64 the shift's draw counter (the next train step draws with this value)      */
  /* Random ensemble mixture head only (num_heads > 0; EINVAL otherwise).  Slots as for the distributional head. */
  B200DQN_NET_PTR_REM_HEADS,        /* (3, batch, A * num_heads) f32 fc2 outputs theta of the last forward           */
  B200DQN_NET_PTR_REM_ALPHAS,       /* (num_heads,) f32 the mixture alpha of the last train step                     */
  B200DQN_NET_PTR_REM_GRADS,        /* (batch, num_heads) f32 gradient dtheta on the taken action's heads            */
  B200DQN_NET_PTR_REM_COUNTER,      /* u64 the mixture's draw counter (the next train step draws with this value)    */
  /* FQF head only (num_fractions > 0; EINVAL otherwise).  The IQN selectors read its rows (N = K = num_fractions,
   * IQN_TAUS holding tauhat) except IQN_TAU_COUNTER, which is EINVAL: the head draws nothing. */
  B200DQN_NET_PTR_FQF_LOGITS,       /* (batch, N) f32 the fraction logits l of the last forward                      */
  B200DQN_NET_PTR_FQF_PROBS,        /* (batch, N) f32 the proposal q                                                 */
  B200DQN_NET_PTR_FQF_FRACTIONS,    /* (batch, N + 1) f32 the fractions tau_0 = 0 .. tau_N = 1                       */
  B200DQN_NET_PTR_FQF_BOUNDARY_QUANTILES, /* (batch (N - 1), A) f32 theta_bnd of the last train step                 */
  B200DQN_NET_PTR_FQF_FRACTION_GRADS,     /* (batch, N - 1) f32 the fraction gradient g of the last train step       */
  B200DQN_NET_PTR_FQF_LOGIT_GRADS,        /* (batch, N) f32 the logit gradient dl of the last train step             */
  /* Bootstrapped heads only (bootstrap_heads > 0; EINVAL otherwise).  REM_HEADS and REM_GRADS read theta and dtheta. */
  B200DQN_NET_PTR_BOOT_MASKS,       /* (batch, K) u8 the bootstrap masks m_k of the last train step                  */
  B200DQN_NET_PTR_BOOT_TARGETS,     /* (batch, K) f32 the per-head targets float(y_k) of the last train step         */
  B200DQN_NET_PTR_BOOT_DELTAS,      /* (batch, K) f32 the per-head TD errors delta_k of the last train step          */
  B200DQN_NET_PTR_BOOT_ACTIVE_HEAD, /* i32 the head predict acts on (-1: the mean over the heads)                    */
  /* Gradient-norm clipping only (max_grad_norm > 0; EINVAL otherwise). */
  B200DQN_NET_PTR_GRAD_SQ,          /* (6,) f64 S_0..S_5, the per-layer sums of squares of the last train step       */
  B200DQN_NET_PTR_GRAD_NORM,        /* f64 N, the global gradient norm of the last train step                         */
  B200DQN_NET_PTR_CLIP_SCALE        /* f32 c32, the clip coefficient of the last train step                           */
};
int b200dqn_net_device_ptr(b200dqn_net* n, int which, void** dev_ptr, size_t* bytes);
/* The tensor-core dgrads write only the fp16 planes of dZ3/dZ2/dZ1; ask them to keep the fp32 copies as well
 * (tests, debugging). */
int b200dqn_net_set_keep_grads(b200dqn_net* n, int keep);
/* Double DQN target (van Hasselt et al., 2016; new capability, no reference counterpart), off by default:
 *   a*_i = argmax_a Q_online(s'_i, a)  (first index of the maximum),  y_i = r_i + discount * Q_target(s'_i, a*_i)
 * in place of max_a Q_target(s'_i, a) (deepqnetwork.py:124,140-143); terminals, reward and error clipping, the cost,
 * the backward and the optimizers are unchanged, and predict is not affected.  The train-step forward runs the online
 * network on the poststates as a third slot of its launches.  The first switch-on allocates that slot's buffers
 * (synchronises the device).  Captured step graphs are rebuilt.  ENOTIMPL once b200dqn_net_comm_init has run;
 * b200dqn_net_comm_init returns ENOTIMPL while it is on.  EINVAL on a net with the Munchausen target. */
int b200dqn_net_set_double_q(b200dqn_net* n, int on);
/* The head predict acts on, on a net with bootstrapped heads: h in 0..K-1 picks head h, h = -1 the mean over the heads.
 * The word lives on the device and is written in stream order: a predict enqueued on `stream` after this call sees h,
 * one enqueued before does not, and a captured fast-path predict graph reads it at every replay.  EINVAL for h outside
 * -1..K-1 and on a net without bootstrapped heads.  Asynchronous. */
int b200dqn_net_set_active_head(b200dqn_net* n, int h, void* stream);
/* Last summed gradient of `layer` converted to NEON layout (tests).  Synchronises. */
int b200dqn_net_get_grads(b200dqn_net* n, int layer, float* host_dW, void* stream);
/* Number of kernels one fused train step launches (bench.py's gpu_launches). */
int b200dqn_net_launches_per_step(const b200dqn_net* n, int* launches);

/* Developer aid: clock64() stamps written by CTA (0,0,0) of the tensor-core kernel whose label equals
 * $B200DQN_TRACE_LABEL (slots documented in csrc/umma2.cuh).  Returns the number of slots or -1. */
int b200dqn_debug_trace(unsigned long long* host_out, int n);

/* ------------------------------------------------------------------ multi-GPU ----------- */

/* Data-parallel learners with replicated replay (SURVEY §8e; new capability, no reference
 * counterpart).  One process per GPU; the 128-byte NCCL unique id is produced on rank 0 and
 * distributed by the host (torch.distributed / a file).  After comm_init every train step
 * all-reduces the summed dW (fp32, 1.69 M elements) over NVLink before the RMSProp update, so
 * weights stay bit-identical on all ranks.  libnccl.so.2 is dlopen()ed at first use (bootstrap,
 * handle exchange, and the fallback data path). */
int b200dqn_comm_unique_id(void* out_id128);
int b200dqn_net_comm_init(b200dqn_net* n, const void* id128, int rank, int world_size);
int b200dqn_net_comm_destroy(b200dqn_net* n);
/* How the gradients travel and whether the exchange is healthy (synchronises the device).
 * *mode: 0 = single learner, 1 = NCCL all-reduce, 2 = peer-memory exchange — every rank maps every
 * other rank's exchange buffers (cudaIpc); fc1's operand rows are gathered with P2P stores so its
 * gradient is never reduced, the small layers use a one-shot LL all-reduce (csrc/comm_p2p.cuh;
 * B200DQN_P2P_SCHED=layer|tail selects the two-shot in-place exchange instead).  Chosen at comm_init
 * when all ranks can map each other, forced off with B200DQN_COMM=nccl.  *error != 0: a peer wait timed out (60 s) since comm_init — the learners
 * are out of step and the results since then are invalid. */
int b200dqn_net_comm_status(b200dqn_net* n, int* mode, int* error);
/* Developer aid (mode 2 only, collective: every rank makes the same call): mean microseconds of `iters`
 * back-to-back in-place exchanges of layers [l0, l1] with the k_xchg switches `flags` and a CTA cap
 * `blocks` (0 = default), and whether one exchange reproduced its known answer.  flags & 16: time the
 * one-shot LL all-reduce of the default schedule instead (l0 == l1, one of layers 0, 1, 2, 4). */
int b200dqn_debug_xchg(b200dqn_net* n, int l0, int l1, int flags, int blocks, int iters, float* us_out, int* ok_out);

#ifdef __cplusplus
}
#endif
#endif /* B200DQN_H */
