// net_umma.cuh — entry points of the tcgen05 (math_mode TCGEN05) engine and of the NCCL glue,
// called from net.cu.
#pragma once
#include <cuda_fp16.h>

#include "common.cuh"
#include "comm_p2p.cuh"
#include "optim.cuh"

struct b200dqn_net;

namespace b200 {

OptArgs make_opt_args(const b200dqn_net* n, int rows);   // net.cu: optimizer constants of this net

// tensor-core engine (net_umma.cu)
int umma_net_init(b200dqn_net* n);                      // allocate operand images etc. (no-op in SIMT mode)
void umma_net_destroy(b200dqn_net* n);
int umma_double_q_alloc(b200dqn_net* n);                // fp16 planes of network slot 2 (Double DQN), once
int umma_weights_changed(b200dqn_net* n, cudaStream_t st);  // fp32 master weights were overwritten by the host
int umma_target_synced(b200dqn_net* n, cudaStream_t st);    // target <- online
// release_early: the launches are links of the single-GPU critical chain; the kernels that gain from it let their
// successor pre-launch right after their own dependency wait
// trunk_only (IQN head): conv1..conv3 only, with the fp32 H3 of slots 0 and 1 kept for the modulation; no fc1
// crop (random_shift): [nb][2] crop offsets of frame sources 0 and 1, or nullptr for unshifted states
int umma_forward(b200dqn_net* n, const uint8_t* const src[2], const int32_t* const idx[2], const int shift[2],
                 const int32_t* const crop[2], int nets, int rows, cudaStream_t st, bool release_early,
                 bool trunk_only = false);
// IQN head: fc1's forward on the modulated rows X (n->d_x16 planes) at `rows` expanded rows with `splits` k-splits
int umma_fc1_fwd_iqn(b200dqn_net* n, int nets, int rows, int splits, cudaStream_t st);
// FQF head: the online network's fc1 forward on the boundary pass's X planes (n->d_bx16) at `rows` rows
int umma_fc1_fwd_fqf_boundary(b200dqn_net* n, int rows, int splits, cudaStream_t st);
int umma_fc1_splits(int rows);
// the Munchausen target pass: the target network on the frames src/idx/shift (the prestates), into slot 2's planes and
// fc1 partials (nets = 1, no fp32 activations); crop: the prestates' crop offsets (slot 0's), or nullptr
int umma_forward_target_pre(b200dqn_net* n, const uint8_t* src, const int32_t* idx, int shift, const int32_t* crop,
                            int rows, cudaStream_t st);
// RMSProp of the fc1 layer + refresh of its tile image in one smem-free kernel; clip (non-null): the update under global
// gradient-norm clipping, with the coefficient c32 read from *clip on the device
int umma_opt_fc1(b200dqn_net* n, int rows, cudaStream_t st, bool from_g = false, const float* clip = nullptr);
// fused split-K reduction + RMSProp + tile-image refresh of conv layer l (0..2), single-GPU tensor-core path
// from_g: read the (all-reduced) gradient from d_g instead of the split-K partials
int umma_opt_conv(b200dqn_net* n, int l, int rows, cudaStream_t st, const char* label, bool from_g = false);
// rebuild the fp16 hi/lo tile images of layers [l0, l1] of network `which` (0 online, 1 target)
int umma_pack_layers(b200dqn_net* n, int which, int l0, int l1, cudaStream_t st);
// soft target update of layer l (0..3): target <- fl(fl(c target) + fl(t online)) and the target's forward image of
// the result, in one pass
int umma_soft_pack(b200dqn_net* n, int l, float c, float t, cudaStream_t st);
// fp16 hi plane of dZ4 and the offset of its lo plane (nullptr when math_mode != TCGEN05)
void umma_dz4_planes(b200dqn_net* n, __half** hi, int64_t* lo_off);
// fp16 hi plane of dZ3 (conv3's output gradient) and the offset of its lo plane (nullptr when math_mode != TCGEN05)
void umma_dz3_planes(b200dqn_net* n, __half** hi, int64_t* lo_off);
int umma_wgrad_splits(int layer, int rows);   // split-K factor of the conv wgrad of `layer` (0..2)
// op: 0 fc1_wgrad, 1 fc1_dgrad, 2 conv3_wgrad, 3 conv3_dgrad, 4 conv2_wgrad, 5 conv2_dgrad, 6 conv1_wgrad
// release_early: as for umma_forward
int umma_backward_op(b200dqn_net* n, int op, const uint8_t* src, const int32_t* idx, int shift, int rows,
                     cudaStream_t st, bool release_early);

// NCCL glue (comm.cu)
int comm_allreduce_grads(b200dqn_net* n, cudaStream_t st);
int comm_allreduce_range(b200dqn_net* n, int l0, int l1, cudaStream_t st);
int comm_xchg_range(b200dqn_net* n, int l0, int l1, int chan, cudaStream_t st, const char* label);
bool comm_gather_active(const b200dqn_net* n, cudaStream_t st);
int comm_xll_layer(b200dqn_net* n, int layer, cudaStream_t st, const char* label);
int comm_xll_args(b200dqn_net* n, int layer, XllArgs* out);   // launch arguments of layer's LL exchange
int umma_opt_conv_xll(b200dqn_net* n, int l, int rows, cudaStream_t st, const char* label);   // experimental, fused
int comm_push_planes(b200dqn_net* n, int chan, const void* hi, int64_t lo_off_elems, cudaStream_t st);
int comm_wait_pushes(b200dqn_net* n, cudaStream_t st, int dz_rows = 0);   // dz_rows > 0: counted head pushes
bool comm_dz4_ll_enabled();
int comm_gather_dz4_ll(b200dqn_net* n, const void* hi, int64_t lo_off_elems, cudaStream_t st, bool wait_h3);   // LL all-gather of the dZ4 planes
bool comm_head_push(const b200dqn_net* n, cudaStream_t st, HeadPush* out);   // gather schedule + head-side dZ4 push on?
// gather schedule hooks of the tensor-core engine (net_umma.cu)
int umma_push_h3(b200dqn_net* n, cudaStream_t st);       // after conv23_fwd: rows of the online net's H3 planes
int umma_push_dz4(b200dqn_net* n, cudaStream_t st);      // after the head
int umma_gather_dz4_ll(b200dqn_net* n, cudaStream_t st); // after the head: LL all-gather of dZ4 (default)
int umma_fc1_wgrad_gathered(b200dqn_net* n, cudaStream_t st);   // dW4 over all world x nb rows
void comm_destroy(b200dqn_net* n);

}  // namespace b200
