"""DeepQNetwork with the reference's call surface (/root/reference/src/deepqnetwork.py:15-192):
the Neon model/train/predict replaced by hand-written sm_90a kernels (csrc/net*.cu)."""
import ctypes as C
import os
import logging
import pickle

import numpy as np

from . import _lib as L
from .replay_memory import DeviceMinibatch
from .state_buffer import DeviceStates

logger = logging.getLogger(__name__)

# (R, S, K, stride) of deepqnetwork.py:83-87
_CONV = [(8, 8, 32, 4), (4, 4, 64, 2), (3, 3, 64, 1)]
# --optimizer (main.py:40, deepqnetwork.py:50-61) -> (library code, number of Neon state arrays per W)
_OPTIMIZERS = {"rmsprop": (L.OPT_RMSPROP, 1), "adam": (L.OPT_ADAM, 2), "adadelta": (L.OPT_ADADELTA, 3)}


def _arg(args, name, default):
    return getattr(args, name, default)


def tau_seed(random_seed):
    """The IQN head's uint64 tau_seed for args.random_seed: a fixed odd multiple of the seed (mod 2^64), so equal seeds
    draw equal taus; a fresh random one when the seed is None."""
    if random_seed is None:
        return int.from_bytes(os.urandom(8), "little")
    return (int(random_seed) * 0x9E3779B97F4A7C15 + 0x632BE59BD9B4E019) % (1 << 64)


def shift_seed(random_seed):
    """The random-shift augmentation's uint64 shift_seed for args.random_seed: like tau_seed, with another odd
    multiplier and offset, so the crops and the IQN head's tau never share a stream; a fresh random one when the seed is
    None."""
    if random_seed is None:
        return int.from_bytes(os.urandom(8), "little")
    return (int(random_seed) * 0xD1B54A32D192ED03 + 0x8CB92BA72F3D8DD7) % (1 << 64)


def rem_seed(random_seed):
    """The REM head's uint64 rem_seed for args.random_seed: like tau_seed and shift_seed, with another odd multiplier
    and offset, so the mixture never shares a stream with them; a fresh random one when the seed is None."""
    if random_seed is None:
        return int.from_bytes(os.urandom(8), "little")
    return (int(random_seed) * 0xA0761D6478BD642F + 0xE7037ED1A0B428DB) % (1 << 64)


def bootstrap_seed(random_seed):
    """The bootstrapped heads' uint64 bootstrap_seed for args.random_seed: like rem_seed, with another odd multiplier and
    offset, so the masks never share a stream with the other draws; a fresh random one when the seed is None."""
    if random_seed is None:
        return int.from_bytes(os.urandom(8), "little")
    return (int(random_seed) * 0xE7037ED1A0B428DB + 0x8EBC6AF09C88C6E3) % (1 << 64)


class DeepQNetwork:
    def __init__(self, num_actions, args, device=None, math_mode=None, stream=None):
        # remember parameters (:17-26)
        self.num_actions = num_actions
        self.batch_size = args.batch_size
        self.discount_rate = args.discount_rate
        self.history_length = args.history_length
        self.screen_dim = (args.screen_height, args.screen_width)
        self.clip_error = args.clip_error
        self.min_reward = args.min_reward
        self.max_reward = args.max_reward
        self.batch_norm = _arg(args, "batch_norm", False)
        # flags of the reference this build accepts but does not implement (SURVEY §8 a17 note)
        if self.batch_norm:
            raise NotImplementedError("--batch_norm is not implemented in this library")
        self.optimizer = _arg(args, "optimizer", "rmsprop")
        assert self.optimizer in _OPTIMIZERS, "Unknown optimizer"       # :60-61
        if np.dtype(_arg(args, "datatype", "float32")) != np.float32:
            raise NotImplementedError("only --datatype float32 is implemented in this library")
        if _arg(args, "stochastic_round", False):
            raise NotImplementedError("--stochastic_round is not implemented in this library")
        if self.clip_error is not None and self.clip_error < 0:
            # the reference hands Neon's be.clip a lower bound above its upper bound (:159), whose result is unpinned
            raise NotImplementedError("--clip_error < 0 is not implemented in this library")
        self.device = _arg(args, "device_id", 0) if device is None else device
        self._stream_obj = stream            # keep the stream alive as long as this object uses it
        self._stream = L.stream_ptr(stream)

        cfg = L.NetConfig()
        L.call("b200dqn_net_config_default", C.byref(cfg), num_actions)
        cfg.batch_size = args.batch_size
        cfg.history_length = args.history_length
        cfg.screen_h, cfg.screen_w = self.screen_dim
        cfg.discount_rate = args.discount_rate
        cfg.learning_rate = args.learning_rate
        cfg.decay_rate = args.decay_rate
        cfg.clip_error = float(args.clip_error or 0)
        cfg.min_reward = float(args.min_reward)         # type=float (main.py:43-44)
        cfg.max_reward = float(args.max_reward)
        cfg.target_steps = int(args.target_steps or 0)
        if math_mode is None:
            math_mode = _arg(args, "math_mode", "fp32")
        cfg.math_mode = {"fp32": L.MATH_FP32_SIMT, "tcgen05": L.MATH_TCGEN05}[math_mode]
        cfg.optimizer, self.num_states = _OPTIMIZERS[self.optimizer]
        self.math_mode = math_mode
        # distributional value head (C51, Bellemare et al., 2017): a new capability, off unless args.distributional is
        # set; it fixes fc2's shape, so it is chosen here and not switchable later
        self.distributional = bool(_arg(args, "distributional", False))
        self.num_atoms, self.support = 0, None
        if self.distributional:
            cfg.num_atoms = int(_arg(args, "num_atoms", 51))
            cfg.v_min = float(_arg(args, "v_min", -10.0))
            cfg.v_max = float(_arg(args, "v_max", 10.0))
        # dueling network (Wang et al., 2016): a new capability, off unless args.dueling is set; it fixes fc1's and fc2's
        # shapes, so it is chosen here and not switchable later
        self.dueling = bool(_arg(args, "dueling", False))
        cfg.dueling = int(self.dueling)
        # quantile-regression value head (QR-DQN, Dabney et al., 2018): a new capability, off unless
        # args.quantile_regression is set; its Huber threshold is clip_error.  Fixed here, like the other heads.
        self.quantile_regression = bool(_arg(args, "quantile_regression", False))
        self.num_quantiles, self.taus = 0, None
        if self.quantile_regression:
            cfg.num_quantiles = int(_arg(args, "num_quantiles", 200))
            assert cfg.num_quantiles >= 1, "num_quantiles %d: the quantile head needs 1..200" % cfg.num_quantiles
        # Munchausen DQN target (Vieillard et al., 2020): a new capability, off unless args.munchausen is set; alpha,
        # tau and the clip l0 default to the paper's 0.9, 0.03 and -1.  It sizes the train step's buffers, so it is
        # fixed here; with args.double_dqn it is refused (AssertionError: the target makes no greedy choice)
        self.munchausen = bool(_arg(args, "munchausen", False))
        if self.munchausen:
            cfg.munchausen = 1
            cfg.munchausen_alpha = float(_arg(args, "munchausen_alpha", 0.9))
            cfg.munchausen_tau = float(_arg(args, "munchausen_tau", 0.03))
            cfg.munchausen_clip = float(_arg(args, "munchausen_clip", -1.0))
        # implicit quantile network head (IQN, Dabney et al., 2018): a new capability, off unless args.implicit_quantiles
        # is set; N = num_tau_samples (64) online and target samples per train row, K = num_quantile_samples (32) per
        # predict row, as Dopamine.  The device draws tau from a hash of tau_seed, derived from random_seed, and a
        # device-resident counter; its embedding is a sixth layer.  Fixed here, like the other heads.
        self.implicit_quantiles = bool(_arg(args, "implicit_quantiles", False))
        self.num_tau_samples = self.num_quantile_samples = 0
        if self.implicit_quantiles:
            cfg.num_tau_samples = int(_arg(args, "num_tau_samples", 64))
            cfg.num_quantile_samples = int(_arg(args, "num_quantile_samples", 32))
            assert cfg.num_tau_samples >= 1, "num_tau_samples %d: the IQN head needs 1..64" % cfg.num_tau_samples
            cfg.tau_seed = tau_seed(_arg(args, "random_seed", None))
        # random-shift augmentation (DrQ, Kostrikov et al., 2020): a new capability, off unless args.random_shift = p > 0
        # (DrQ uses 4).  Every train step trains on states padded by p with their edge pixels and cropped back to
        # 84x84 at offsets the device draws from shift_seed, derived from random_seed, and a device-resident counter.
        # predict and the stored frames are never shifted.
        self.random_shift = int(_arg(args, "random_shift", 0))
        if self.random_shift:
            cfg.random_shift = self.random_shift
            cfg.shift_seed = self.shift_seed = shift_seed(_arg(args, "random_seed", None))
        # random ensemble mixture head (REM, Agarwal et al., 2020): a new capability, off unless args.rem is set; K =
        # num_heads (200) Q-value heads per action, mixed in each train step by a convex combination the device draws
        # from rem_seed, derived from random_seed, and a device-resident counter; predict takes the mean over the heads.
        # Fixed here, like the other heads.
        self.rem = bool(_arg(args, "rem", False))
        self.num_heads = 0
        if self.rem:
            cfg.num_heads = int(_arg(args, "num_heads", 200))
            assert cfg.num_heads >= 1, "num_heads %d: the REM head needs 1..200" % cfg.num_heads
            cfg.rem_seed = self.rem_seed = rem_seed(_arg(args, "random_seed", None))
        # fully parameterized quantile function head (FQF, Yang et al., 2019): a new capability, off unless args.fqf is
        # set; N = num_fractions (32) fractions per sample, proposed from the online network's conv3 output by a seventh
        # layer W_f trained at fraction_lr (this project's default 2.5e-9).  It is an IQN net whose tau is the proposal
        # (no draw, no seed).  Fixed here, like the other heads.
        self.fqf = bool(_arg(args, "fqf", False))
        self.num_fractions = 0
        if self.fqf:
            cfg.num_fractions = int(_arg(args, "num_fractions", 32))
            cfg.fraction_lr = float(_arg(args, "fraction_lr", 2.5e-9))
            assert cfg.num_fractions >= 2, "num_fractions %d: the FQF head needs 2..64" % cfg.num_fractions
        # bootstrapped DQN heads (Osband et al., 2016): a new capability, off unless args.bootstrapped is set; K =
        # bootstrap_heads (10) Q-value heads per action on the shared network, each trained on its own target with a
        # Bernoulli(bootstrap_p) mask (0.5) the device hashes from bootstrap_seed, derived from random_seed, and the
        # transition's ring slot.  predict acts on the active head (set_active_head / sample_head), or on the mean over
        # the heads (-1, the default).  Fixed here, like the other heads.
        self.bootstrapped = bool(_arg(args, "bootstrapped", False))
        if self.bootstrapped:
            cfg.bootstrap_heads = int(_arg(args, "bootstrap_heads", 10))
            cfg.bootstrap_p = float(_arg(args, "bootstrap_p", 0.5))
            assert cfg.bootstrap_heads >= 1, "bootstrap_heads %d: bootstrapped heads need 1..200" % cfg.bootstrap_heads
            cfg.bootstrap_seed = self.bootstrap_seed = bootstrap_seed(_arg(args, "random_seed", None))
        # soft (Polyak-averaged) target update: a new capability, off unless args.soft_target_tau = tau > 0 (SB3's and
        # CleanRL's `tau`; BBF uses 0.005).  Every train step ends with target <- (1 - tau) target + tau online on the
        # device; update_target_network() keeps its hard copy.  It needs a separate target network (target_steps > 0).
        cfg.soft_target_tau = float(_arg(args, "soft_target_tau", 0.0) or 0.0)
        self.soft_target_tau = cfg.soft_target_tau
        # global gradient-norm clipping: a new capability, off unless args.max_grad_norm = M > 0 (SB3's name; SB3 uses
        # 10, as do OpenAI baselines' Atari DQN and the dueling paper).  Every train step scales the whole update by
        # min(1, M / (||g / bsz|| + 1e-6)) on the device (b200dqn.h states the rule).  Fixed at creation.
        cfg.max_grad_norm = float(_arg(args, "max_grad_norm", 0.0) or 0.0)
        self.max_grad_norm = cfg.max_grad_norm or None
        h = C.c_void_p()
        L.call("b200dqn_net_create", self.device, C.byref(cfg), C.byref(h))
        self._h = h
        if self.distributional:
            self.num_atoms, self.v_min, self.v_max = cfg.num_atoms, cfg.v_min, cfg.v_max
            dz = (cfg.v_max - cfg.v_min) / (cfg.num_atoms - 1)         # z_i = v_min + i dz in fp64, as the device
            self.support = np.array([cfg.v_min + i * dz for i in range(cfg.num_atoms)], dtype=np.float64)
        if self.implicit_quantiles:
            self.num_tau_samples, self.num_quantile_samples = cfg.num_tau_samples, cfg.num_quantile_samples
            self.tau_seed = cfg.tau_seed
        if self.rem:
            self.num_heads = cfg.num_heads
        if self.bootstrapped:   # the REM head's fc2 and readers, K = bootstrap_heads
            self.num_heads, self.bootstrap_p = cfg.bootstrap_heads, cfg.bootstrap_p
            self._head_rng = np.random.RandomState(self.bootstrap_seed % (1 << 32))
        if self.fqf:   # the IQN accessors read its rows: N = K = num_fractions
            self.num_fractions = self.num_tau_samples = self.num_quantile_samples = cfg.num_fractions
            self.fraction_lr = cfg.fraction_lr
        if self.quantile_regression:
            self.num_quantiles = n = cfg.num_quantiles                 # tau_i = (2i + 1) / 2N in fp64, as the device
            self.taus = np.array([(2 * i + 1) / (2 * n) for i in range(n)], dtype=np.float64).astype(np.float32)

        # model.initialize (:49, :70): Xavier draws from one numpy RandomState(random_seed) —
        # online layers first, then the separately-initialised target model.  An IQN embedding is drawn after fc2 of
        # its network, with fan_in 64.  The FQF fraction layer takes no draw and stays zero: the first proposal is
        # uniform, and layers 0-5 are drawn as on an IQN net.
        rng = np.random.RandomState(_arg(args, "random_seed", None))
        for which in ((0, 1) if cfg.target_steps else (0,)):
            for layer, shp in enumerate(self.layer_shapes()[:6]):
                fan_in = shp[0] if layer < 3 else shp[1]               # Xavier(local=True / False) (:79-80)
                scale = np.sqrt(3.0 / fan_in)
                w = rng.uniform(-scale, scale, shp).astype(np.float32)
                self._set_layer(which, layer, w, np.zeros_like(w))
        self.train_iterations = 0
        # Double DQN target (van Hasselt et al., 2016): a new capability, off unless args.double_dqn is set
        self.double_dqn = False
        if _arg(args, "double_dqn", False):
            self.set_double_dqn(True)
        self.save_weights_prefix = _arg(args, "save_weights_prefix", None)
        self.callback = None

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            try:
                L.load().b200dqn_net_destroy(h)
            except Exception:
                pass

    # ---- weights in Neon layout
    def layer_shapes(self):
        out = []
        for layer in range(7 if self.fqf else 6 if self.implicit_quantiles else 5):
            r, c = C.c_int(), C.c_int()
            L.call("b200dqn_net_layer_shape", self._h, layer, C.byref(r), C.byref(c))
            out.append((r.value, c.value))
        return out

    def _set_layer(self, which, layer, w, s=None):
        w = np.ascontiguousarray(w, dtype=np.float32)
        s = None if s is None else np.ascontiguousarray(s, dtype=np.float32)
        assert w.shape == self.layer_shapes()[layer], (w.shape, self.layer_shapes()[layer])
        L.call("b200dqn_net_set_weights", self._h, which, layer, L.np_ptr(w), L.np_ptr(s), self._stream)

    def set_weights(self, weights, states=None, which=0):
        """states: per layer either ONE array (Neon's ``states[0]``, all RMSProp needs) or the list of the
        optimizer's state arrays (Adam [m, v], Adadelta [E[g^2], E[dx^2], dx])."""
        for layer, w in enumerate(weights):
            st = None if states is None else states[layer]
            if isinstance(st, (list, tuple)):
                self._set_layer(which, layer, w, None)
                self._set_states(which, layer, st)
            else:
                self._set_layer(which, layer, w, st)

    def _set_states(self, which, layer, arrays):
        assert len(arrays) <= self.num_states, (len(arrays), self.num_states)
        for k, a in enumerate(arrays):
            a = np.ascontiguousarray(a, dtype=np.float32)
            assert a.shape == self.layer_shapes()[layer]
            L.call("b200dqn_net_set_state", self._h, which, layer, k, L.np_ptr(a), self._stream)

    def get_weights(self, which=0, with_states=True):
        ws, ss = [], []
        for layer, shp in enumerate(self.layer_shapes()):
            w = np.empty(shp, dtype=np.float32)
            s = np.empty(shp, dtype=np.float32) if with_states else None
            L.call("b200dqn_net_get_weights", self._h, which, layer, L.np_ptr(w), L.np_ptr(s), self._stream)
            ws.append(w)
            ss.append(s)
        return (ws, ss) if with_states else ws

    def get_states(self, which=0):
        """Every optimizer state array per layer, like Neon's ``states`` lists."""
        out = []
        for layer, shp in enumerate(self.layer_shapes()):
            planes = []
            for k in range(self.num_states):
                a = np.empty(shp, dtype=np.float32)
                L.call("b200dqn_net_get_state", self._h, which, layer, k, L.np_ptr(a), self._stream)
                planes.append(a)
            out.append(planes)
        return out

    def keep_grads(self, keep=True):
        """Make the tensor-core dgrads also write the fp32 dZ3/dZ2/dZ1 next to their fp16 planes (tests / debugging)."""
        L.call("b200dqn_net_set_keep_grads", self._h, int(bool(keep)))

    def set_double_dqn(self, on=True):
        """Switch the Double DQN target on or off: the online network picks the poststate action (first index of the
        maximum), the target network values it.  Raises NotImplementedError for data-parallel learners."""
        L.call("b200dqn_net_set_double_q", self._h, int(bool(on)))
        self.double_dqn = bool(on)

    def get_grads(self):
        out = []
        for layer, shp in enumerate(self.layer_shapes()):
            g = np.empty(shp, dtype=np.float32)
            L.call("b200dqn_net_get_grads", self._h, layer, L.np_ptr(g), self._stream)
            out.append(g)
        return out

    def device_view(self, which, shape):
        p, b = C.c_void_p(), C.c_size_t()
        L.call("b200dqn_net_device_ptr", self._h, which, C.byref(p), C.byref(b))
        return L.DeviceArray(p.value, shape, "<f4", owner=self)

    def _read_f32(self, which, shape):
        return L.download(self.device, self.device_view(which, shape).ptr, shape, np.float32, self._stream)

    def _read_clip(self, which, shape, dtype):
        if not self.max_grad_norm:
            raise ValueError("the net has no gradient-norm clipping (max_grad_norm)")
        return L.download(self.device, self.device_view(which, shape).ptr, shape, dtype, self._stream)

    def last_grad_sq(self):
        """(6,) float64 per-layer sums of squares S_l of g / bsz of the last train step (layer 5: the embedding)."""
        return self._read_clip(L.NET_PTR_GRAD_SQ, (6,), np.float64)

    def last_grad_norm(self):
        """The global gradient norm N (float64) of the last train step."""
        return float(self._read_clip(L.NET_PTR_GRAD_NORM, (1,), np.float64)[0])

    def last_clip_scale(self):
        """The clip coefficient c32 (float32) the last train step scaled its update by."""
        return self._read_clip(L.NET_PTR_CLIP_SCALE, (1,), np.float32)[0]

    def last_q(self):
        """(preq, postq) of the last train() as (batch, A) arrays (deepqnetwork.py:120,129)."""
        shp = (self.batch_size, self.num_actions)
        return self._read_f32(L.NET_PTR_Q_ONLINE, shp), self._read_f32(L.NET_PTR_Q_TARGET, shp)

    def last_activations(self):
        """Online-network activations of the last forward as NCHW arrays like the oracle's."""
        b = self.batch_size
        h1 = self._read_f32(L.NET_PTR_H1, (b, 20, 20, 32)).transpose(0, 3, 1, 2)
        h2 = self._read_f32(L.NET_PTR_H2, (b, 9, 9, 64)).transpose(0, 3, 1, 2)
        h3 = self._read_f32(L.NET_PTR_H3, (b, 7, 7, 64)).transpose(0, 3, 1, 2)
        h4 = self._read_f32(L.NET_PTR_H4, (b, self._hidden()))
        return h1, h2, h3, h4

    def last_dz(self):
        """Online-network gradients at the pre-activations of the last train() as NCHW arrays (dZ1, dZ2, dZ3, dZ4),
        Rectlin masks applied.  On the tensor-core engine dZ1..dZ3 are only written while keep_grads() is on."""
        b = self.batch_size
        dz1 = self._read_f32(L.NET_PTR_DZ1, (b, 20, 20, 32)).transpose(0, 3, 1, 2)
        dz2 = self._read_f32(L.NET_PTR_DZ2, (b, 9, 9, 64)).transpose(0, 3, 1, 2)
        dz3 = self._read_f32(L.NET_PTR_DZ3, (b, 7, 7, 64)).transpose(0, 3, 1, 2)
        dz4 = self._read_f32(L.NET_PTR_DZ4, (b, self._hidden()))
        return dz1, dz2, dz3, dz4

    def _hidden(self):
        return self.layer_shapes()[3][0]                                # fc1's width: 512, or 1024 on a dueling net

    def last_dz4_planes(self):
        """(hi, lo) float16 planes of dZ4 the tensor-core dgrad reads, each (batch, 512), or (batch, 1024) on a dueling
        net; lo is scaled by 2048."""
        p, b = C.c_void_p(), C.c_size_t()
        L.call("b200dqn_net_device_ptr", self._h, L.NET_PTR_DZ4_PLANES, C.byref(p), C.byref(b))
        shape = (self.batch_size, self._hidden())
        lo_off = b.value // 2 - shape[0] * shape[1]
        hi = L.download(self.device, p.value, shape, np.float16, self._stream)
        lo = L.download(self.device, p.value + 2 * lo_off, shape, np.float16, self._stream)
        return hi, lo

    def last_online_postq(self):
        """The online network's Q on the poststates of the last Double DQN train() as a (batch, A) array."""
        return self._read_f32(L.NET_PTR_Q_ONLINE_POST, (self.batch_size, self.num_actions))

    def last_td_errors(self):
        """TD errors before the clip of the last train() on a prioritized ring, (batch,) float32."""
        return self._read_f32(L.NET_PTR_TD_ERRORS, (self.batch_size,))

    def last_row_costs(self):
        """Per-sample costs of the last train() (before the clip, importance-weighted on a prioritized ring), (batch,)
        float32; the step's cost is their mean, summed in row order."""
        return self._read_f32(L.NET_PTR_ROW_COSTS, (self.batch_size,))

    def last_deltas(self):
        return self._read_f32(L.NET_PTR_DELTAS, (self.batch_size, self.num_actions))

    # ---- distributional head (num_atoms > 0): slot 0 online on the prestates, 1 target on the poststates, 2 online on
    # the poststates (Double DQN)
    def last_logits(self):
        """fc2's outputs of the last forward, (3, batch, A, num_atoms) float32."""
        return self._read_f32(L.NET_PTR_LOGITS, (3, self.batch_size, self.num_actions, self.num_atoms))

    def last_distributions(self):
        """Softmax of each action's logits of the last forward, (3, batch, A, num_atoms) float32."""
        return self._read_f32(L.NET_PTR_PROBS, (3, self.batch_size, self.num_actions, self.num_atoms))

    def last_target_distribution(self):
        """The projected target distribution m of the last train(), (batch, num_atoms) float32."""
        return self._read_f32(L.NET_PTR_TARGET_DIST, (self.batch_size, self.num_atoms))

    def last_logit_grads(self):
        """The gradient on the taken action's logits of the last train(), (batch, num_atoms) float32."""
        return self._read_f32(L.NET_PTR_LOGIT_GRADS, (self.batch_size, self.num_atoms))

    # ---- quantile-regression head (num_quantiles > 0): slots as for the distributional head
    def last_quantiles(self):
        """fc2's outputs theta of the last forward, (3, batch, A, num_quantiles) float32."""
        return self._read_f32(L.NET_PTR_QUANTILES, (3, self.batch_size, self.num_actions, self.num_quantiles))

    def last_target_quantiles(self):
        """The target quantiles T_j of the last train(), (batch, num_quantiles) float32."""
        return self._read_f32(L.NET_PTR_TARGET_QUANTILES, (self.batch_size, self.num_quantiles))

    def last_quantile_grads(self):
        """The gradient on the taken action's quantiles of the last train(), (batch, num_quantiles) float32."""
        return self._read_f32(L.NET_PTR_QUANTILE_GRADS, (self.batch_size, self.num_quantiles))

    # ---- implicit quantile network head (implicit_quantiles = True).  Rows r = b * N + j of the last train(), slot 0
    # online on the prestates and slot 1 target on the poststates; after a predict, slot 0 holds rows b * K + k.
    def last_taus(self):
        """tau of the last forward, (2, batch * max(N, K)) float32."""
        return self._read_f32(L.NET_PTR_IQN_TAUS, (2, self._iqn_rows()))

    def last_iqn_quantiles(self):
        """fc2's outputs theta of the last forward, (2, batch * max(N, K), A) float32."""
        return self._read_f32(L.NET_PTR_IQN_QUANTILES, (2, self._iqn_rows(), self.num_actions))

    def last_iqn_target_quantiles(self):
        """The target quantiles T_j of the last train(), (batch, N) float32."""
        return self._read_f32(L.NET_PTR_IQN_TARGET_QUANTILES, (self.batch_size, self.num_tau_samples))

    def last_iqn_quantile_grads(self):
        """The gradient dtheta on the taken action of each online row of the last train(), (batch, N) float32."""
        return self._read_f32(L.NET_PTR_IQN_QUANTILE_GRADS, (self.batch_size, self.num_tau_samples))

    # ---- fully parameterized quantile function head (fqf = True).  Its rows are the IQN head's at N = K = num_fractions:
    # last_taus() holds tauhat
    def last_fraction_logits(self):
        """The fraction logits l of the last forward, (batch, N) float32."""
        return self._read_f32(L.NET_PTR_FQF_LOGITS, (self.batch_size, self.num_fractions))

    def last_fraction_probs(self):
        """The proposal q = softmax(l) of the last forward, (batch, N) float32."""
        return self._read_f32(L.NET_PTR_FQF_PROBS, (self.batch_size, self.num_fractions))

    def last_fractions(self):
        """The fractions tau_0 = 0 < ... < tau_N = 1 of the last forward, (batch, N + 1) float32."""
        return self._read_f32(L.NET_PTR_FQF_FRACTIONS, (self.batch_size, self.num_fractions + 1))

    def last_boundary_quantiles(self):
        """The online network's theta at tau_1..tau_{N-1} of the last train(), (batch, N - 1, A) float32."""
        return self._read_f32(L.NET_PTR_FQF_BOUNDARY_QUANTILES,
                              (self.batch_size, self.num_fractions - 1, self.num_actions))

    def last_fraction_grads(self):
        """The fraction gradient g_1..g_{N-1} of the last train(), (batch, N - 1) float32."""
        return self._read_f32(L.NET_PTR_FQF_FRACTION_GRADS, (self.batch_size, self.num_fractions - 1))

    def last_fraction_logit_grads(self):
        """The logit gradient dl of the last train(), (batch, N) float32."""
        return self._read_f32(L.NET_PTR_FQF_LOGIT_GRADS, (self.batch_size, self.num_fractions))

    def _iqn_rows(self):
        return self.batch_size * max(self.num_tau_samples, self.num_quantile_samples)

    # ---- random-shift augmentation (random_shift = p > 0)
    def last_shifts(self):
        """The crop offsets (dy, dx) of the last train step, (2, batch, 2) int32: slot 0 the prestates, slot 1 the
        poststates.  Shifted pixel (y, x) is stored pixel (clip(y + dy, 0, 83), clip(x + dx, 0, 83))."""
        return L.download(self.device, self.device_view(L.NET_PTR_SHIFT_OFFSETS, (2, self.batch_size, 2)).ptr,
                          (2, self.batch_size, 2), np.int32, self._stream)

    def shift_draws(self):
        """The shift's draw counter: train steps that have drawn offsets; the next one draws with this value."""
        return int(L.download(self.device, self.device_view(L.NET_PTR_SHIFT_DRAWS, (1,)).ptr, (1,), np.uint64,
                              self._stream)[0])

    # ---- random ensemble mixture head (rem = True): slots as for the distributional head
    def last_heads(self):
        """fc2's outputs theta of the last forward, (3, batch, A, num_heads) float32."""
        return self._read_f32(L.NET_PTR_REM_HEADS, (3, self.batch_size, self.num_actions, self.num_heads))

    def last_mixture(self):
        """The mixture alpha of the last train step, (num_heads,) float32: positive, summing to 1."""
        return self._read_f32(L.NET_PTR_REM_ALPHAS, (self.num_heads,))

    def last_head_grads(self):
        """The gradient on the taken action's heads of the last train(), (batch, num_heads) float32."""
        return self._read_f32(L.NET_PTR_REM_GRADS, (self.batch_size, self.num_heads))

    def mixture_counter(self):
        """The mixture's draw counter: train steps that have drawn alpha; the next one draws with this value."""
        return int(L.download(self.device, self.device_view(L.NET_PTR_REM_COUNTER, (1,)).ptr, (1,), np.uint64,
                              self._stream)[0])

    # ---- bootstrapped heads (bootstrapped = True); last_heads() and last_head_grads() read theta and dtheta
    @property
    def active_head(self):
        """The head predict acts on, read from the device: 0..K-1, or -1 for the mean over the heads."""
        return int(L.download(self.device, self.device_view(L.NET_PTR_BOOT_ACTIVE_HEAD, (1,)).ptr, (1,), np.int32,
                              self._stream)[0])

    def set_active_head(self, h):
        """Act on head h (0..K-1), or on the mean over the heads (-1): every predict issued after this call."""
        L.call("b200dqn_net_set_active_head", self._h, int(h), self._stream)

    def sample_head(self):
        """Draw the next episode's head uniformly from this net's own RandomState and act on it; returns it."""
        assert self.bootstrapped, "sample_head needs bootstrapped heads"
        h = int(self._head_rng.randint(self.num_heads))
        self.set_active_head(h)
        return h

    def last_bootstrap_masks(self):
        """The bootstrap masks of the last train step, (batch, K) uint8."""
        return L.download(self.device, self.device_view(L.NET_PTR_BOOT_MASKS, (1,)).ptr,
                          (self.batch_size, self.num_heads), np.uint8, self._stream)

    def last_head_targets(self):
        """The per-head targets float(y_k) of the last train step, (batch, K) float32."""
        return self._read_f32(L.NET_PTR_BOOT_TARGETS, (self.batch_size, self.num_heads))

    def last_head_deltas(self):
        """The per-head TD errors delta_k of the last train step, (batch, K) float32."""
        return self._read_f32(L.NET_PTR_BOOT_DELTAS, (self.batch_size, self.num_heads))

    # ---- Munchausen target (munchausen = True)
    def last_target_q_pre(self):
        """The target network's Q on the prestates of the last train(), (batch, A) float32: the row whose log-policy
        at the taken action forms the Munchausen bonus (with target_steps = 0 the online row, last_q()[0])."""
        return self._read_f32(L.NET_PTR_Q_TARGET_PRE, (self.batch_size, self.num_actions))

    def last_td_targets(self):
        """The Munchausen targets float(y) of the last train(), (batch,) float32."""
        return self._read_f32(L.NET_PTR_TD_TARGETS, (self.batch_size,))

    # ---- dueling network: slots as for the distributional head
    def last_advantages(self):
        """The advantage stream's outputs A_a of the last forward, (3, batch, A) float32."""
        return self._read_f32(L.NET_PTR_DUELING_VA, (3, self.batch_size, self.num_actions + 1))[..., :-1]

    def last_values(self):
        """The value stream's output V of the last forward, (3, batch) float32."""
        return self._read_f32(L.NET_PTR_DUELING_VA, (3, self.batch_size, self.num_actions + 1))[..., -1]

    # ---- reference methods
    def update_target_network(self, tau=None):
        """tau None: the reference's hard copy of the online network, optimizer states included (:102-105).  A float
        tau in (0, 1]: one soft update, target <- (1 - tau) target + tau online, weights only (the interval form of the
        soft target update, a blend every k-th train step)."""
        if tau is None:
            L.call("b200dqn_net_sync_target", self._h, self._stream)    # :102-105
        else:
            L.call("b200dqn_net_soft_update_target", self._h, float(tau), self._stream)

    def train(self, minibatch, epoch=0):
        """deepqnetwork.py:107-172.  A pristine DeviceMinibatch is trained in place from the ring, and so is one from a
        prioritized or n-step ring even once it has been looked at (the importance weights, the priority update and
        the n-step window live there), and so is every one on a net with bootstrapped heads at bootstrap_p < 1 (the
        masks belong to the ring slots).  A host tuple is always the uniform, unweighted one-step step, and such a net
        refuses it (NotImplementedError)."""
        ring_masks = self.bootstrapped and self.bootstrap_p < 1
        if isinstance(minibatch, DeviceMinibatch) and (not minibatch.materialised or minibatch._mem.prioritized or
                                                       minibatch._mem.n_step > 1 or ring_masks):
            minibatch._check_current()
            mem = minibatch._mem
            cost = C.c_float()
            if not minibatch.sampled:
                # the index draw rides in this step's graph: one launch, results through host-mapped memory
                words = C.c_uint32()
                lockstep = mem.rng_mode == "python"
                key, pos = mem._host_upload_args() if lockstep else (None, 0)
                if not lockstep and not mem._rng_on_device:
                    mem.seed_device_rng()
                want = lockstep or self.callback is not None
                L.call("b200dqn_net_step_host", self._h, mem._h, 0, None, None, None, None, 1, key, pos,
                       C.byref(cost) if want else None, C.byref(words) if lockstep else None, self._stream)
                minibatch.sampled = True
                if lockstep:
                    mem._host_advance(words.value)
                self.train_iterations += 1
                if self.callback:
                    self.callback.on_train(np.float32(cost.value))      # :171-172 (cost[0,0] is a numpy float32)
            elif self.callback:
                L.call("b200dqn_net_train_sampled_cost", self._h, mem._h, C.byref(cost), self._stream)
                self.train_iterations += 1
                self.callback.on_train(np.float32(cost.value))          # :171-172
            else:
                L.call("b200dqn_net_train_sampled", self._h, mem._h, self._stream)
                self.train_iterations += 1
            return
        prestates, actions, rewards, poststates, terminals = minibatch
        assert len(prestates.shape) == 4                                # :110-116
        assert len(poststates.shape) == 4
        assert len(actions.shape) == 1
        assert len(rewards.shape) == 1
        assert len(terminals.shape) == 1
        assert prestates.shape == poststates.shape
        assert prestates.shape[0] == actions.shape[0] == rewards.shape[0] == poststates.shape[0] == terminals.shape[0]
        assert prestates.shape == (self.batch_size, self.history_length) + self.screen_dim
        pre = np.ascontiguousarray(prestates, dtype=np.uint8)
        post = np.ascontiguousarray(poststates, dtype=np.uint8)
        act = np.ascontiguousarray(actions, dtype=np.uint8)
        rew = np.ascontiguousarray(rewards, dtype=np.int64)
        term = np.ascontiguousarray(terminals, dtype=np.uint8)
        cost = C.c_float()
        L.call("b200dqn_net_train", self._h, L.np_ptr(pre), L.np_ptr(act), L.np_ptr(rew), L.np_ptr(post),
               L.np_ptr(term), C.byref(cost), self._stream)
        self.train_iterations += 1                                      # :168
        if self.callback:
            self.callback.on_train(np.float32(cost.value))              # :171-172 (cost[0,0] is a numpy float32)

    def train_fused(self, mem, nsteps=1):
        """`nsteps` x (mem.getMinibatch(); self.train(...)) of agent.py:112-114 with no host round trip
        (device-resident MT19937 stream).  Costs stay on the device — see :meth:`last_costs`."""
        if not mem._rng_on_device:
            mem.seed_device_rng()
        L.call("b200dqn_net_train_fused", self._h, mem._h, int(nsteps), self._stream)
        self.train_iterations += nsteps
        mem._sample_ticket += nsteps
        mem._host_state_in_sync = None        # the device stream ran ahead of the host's `random`

    def step_host(self, mem, actions, rewards, screens, terminals, train_repeat=1):
        """agent.py:102-114 for a caller that owns the loop, as ONE library call: the (action, reward, screen,
        terminal) of the env steps since the last train are appended to `mem`, then `train_repeat` x
        (mem.getMinibatch(); self.train(...)) run on the device.  With ``mem.rng_mode == "python"`` the process-global
        `random` stays in lock-step (state up if it moved, words consumed back).  Returns the costs (float32 array)
        and delivers them to ``callback.on_train`` in order, like the reference's per-train callback."""
        n = len(actions)
        a = np.ascontiguousarray(actions, dtype=np.uint8)
        r = np.ascontiguousarray(rewards, dtype=np.int64)
        s = np.ascontiguousarray(screens, dtype=np.uint8)
        t = np.ascontiguousarray(terminals, dtype=np.uint8)
        assert s.shape == (n,) + tuple(mem.dims) and a.shape == r.shape == t.shape == (n,)
        costs = np.zeros(max(train_repeat, 1), dtype=np.float32)
        words = C.c_uint32()
        lockstep = mem.rng_mode == "python"
        key, pos = mem._host_upload_args() if (lockstep and train_repeat) else (None, 0)
        if not lockstep and not mem._rng_on_device:
            mem.seed_device_rng()
        L.call("b200dqn_net_step_host", self._h, mem._h, n, L.np_ptr(a), L.np_ptr(r), L.np_ptr(s), L.np_ptr(t),
               int(train_repeat), key, pos, L.np_ptr(costs) if train_repeat else None,
               C.byref(words) if (lockstep and train_repeat) else None, self._stream)
        if train_repeat:
            mem._sample_ticket += train_repeat
            if lockstep:
                mem._host_advance(words.value)
            else:
                mem._host_state_in_sync = None
            for c in costs[:train_repeat]:
                self.train_iterations += 1
                if self.callback:
                    self.callback.on_train(np.float32(c))
        return costs[:train_repeat]

    def last_costs(self, count=1):
        out = np.empty(count, dtype=np.float32)
        L.call("b200dqn_net_read_costs", self._h, int(count), L.np_ptr(out), self._stream)
        return out

    def predict(self, states):
        # :176 — the minibatch is full size
        assert tuple(states.shape) == ((self.batch_size, self.history_length,) + self.screen_dim)
        q = np.empty((self.batch_size, self.num_actions), dtype=np.float32)
        if isinstance(states, DeviceStates):
            # one graph launch, Q row(s) back through host-mapped memory (agent.py:55-61 runs this every env step)
            L.call("b200dqn_net_predict_device_host", self._h, C.c_void_p(states.device_ptr()), states.live_rows,
                   L.np_ptr(q), self._stream)
            return q
        st = np.ascontiguousarray(states, dtype=np.uint8)
        L.call("b200dqn_net_predict", self._h, L.np_ptr(st), L.np_ptr(q), self._stream)
        return q                                                        # (batch, A) == qvalues.T (:186)

    def load_weights(self, load_path):
        """Model.load_params (:188-189): both pickle layouts found in the reference's snapshots/ —
        the pre-1.0 ``layer_params_states`` list (breakout/pong; src/util/convert_weights.py:10-12) and the
        neon-1.3.0 ``model.config.layers`` list (seaquest/space_invaders).  Weights AND optimizer states
        are restored (Model.load_params(load_states=True) is Neon's default)."""
        with open(load_path, "rb") as f:
            d = pickle.load(f, encoding="latin1")
        if "layer_params_states" in d:
            ls = d["layer_params_states"]
        else:
            ls = [l for l in d["model"]["config"]["layers"] if "params" in l]
        if self.fqf:
            assert len(ls) == 7, ("checkpoint holds %d weight layers; an FQF net needs seven: the five of "
                                  "deepqnetwork.py:77-92, the tau embedding and the fraction layer" % len(ls))
        elif self.implicit_quantiles:
            assert len(ls) == 6, ("checkpoint holds %d weight layers; an IQN net needs six: the five of "
                                  "deepqnetwork.py:77-92 and the tau embedding" % len(ls))
        else:
            assert len(ls) == 5, "checkpoint does not hold the five weight layers of deepqnetwork.py:77-92"
        ws = [np.asarray(l["params"]["W"], dtype=np.float32) for l in ls]
        for layer, (l, w) in enumerate(zip(ls, ws)):
            assert w.shape == self.layer_shapes()[layer], \
                "layer %d: checkpoint shape %s, network shape %s" % (layer, w.shape, self.layer_shapes()[layer])
            st = [np.asarray(a, dtype=np.float32) for a in (l.get("states") or [])][:self.num_states]
            self._set_layer(0, layer, w, None)
            if st:
                self._set_states(0, layer, st)
            if len(st) < self.num_states:        # states the checkpoint's optimizer did not keep start at zero
                self._set_states(0, layer, st + [np.zeros_like(w)] * (self.num_states - len(st)))

    def save_weights(self, save_path, layout="neon-1.3.0"):
        """Model.save_params (:191-192).  ``layout="neon-1.3.0"`` (default) writes the structure the reference's
        current Neon writes and reads (same keys, layer list and type strings as snapshots/seaquest_178.pkl);
        ``layout="pre-1.0"`` writes the older ``layer_params_states`` list.  :meth:`load_weights` reads both."""
        ws = self.get_weights(with_states=False)
        ss = self.get_states()
        if layout == "pre-1.0":
            d = {"epoch_index": 0,
                 "layer_params_states": [{"params": {"W": w}, "states": list(s)} for w, s in zip(ws, ss)]}
        else:
            assert layout == "neon-1.3.0", layout
            layers = []
            for i, (w, s) in enumerate(zip(ws, ss)):
                if i < 3:
                    r, _, k, stride = _CONV[i]
                    layers.append({"type": "neon.layers.layer.Convolution",
                                   "config": {"fshape": (r, r, k), "strides": stride, "name": "Convolution_%d" % i,
                                              "parallelism": "Disabled",
                                              "init": {"type": "neon.initializers.initializer.Xavier",
                                                       "config": {"local": True}}},
                                   "params": {"W": w}, "states": list(s)})
                else:
                    layers.append({"type": "neon.layers.layer.Linear",
                                   "config": {"nout": int(w.shape[0]), "name": "Linear_%d" % (i - 3),
                                              "init": {"type": "neon.initializers.initializer.Xavier",
                                                       "config": {"local": False}}},
                                   "params": {"W": w}, "states": list(s)})
                if i < 4:                                            # Rectlin after the first four (:83-89)
                    name = layers[-1]["config"]["name"]
                    layers.append({"type": "neon.layers.layer.Activation",
                                   "config": {"name": name + "_Rectlin",
                                              "transform": {"type": "neon.transforms.activation.Rectlin",
                                                            "config": {"name": "Rectlin_%d" % i}}}})
            d = {"neon_version": "1.3.0+344372b", "epoch_index": 0,
                 "train_input_shape": (self.history_length,) + self.screen_dim,
                 "backend": {"type": "b200dqn", "compat_mode": "neon", "rng_seed": None},
                 "cost": {"type": "neon.layers.layer.GeneralizedCost",
                          "config": {"name": "GeneralizedCost_0",
                                     "costfunc": {"type": "neon.transforms.cost.SumSquared", "config": {}}}},
                 "model": {"type": "neon.layers.container.Sequential", "container": True,
                           "config": {"name": "Sequential_0", "layers": layers}}}
        with open(save_path, "wb") as f:
            pickle.dump(d, f, protocol=2)

    # ---- multi-GPU (new capability, SURVEY §8e)
    def comm_init(self, unique_id, rank, world_size):
        buf = (C.c_char * 128).from_buffer_copy(bytes(unique_id))
        L.call("b200dqn_net_comm_init", self._h, buf, rank, world_size)

    def comm_destroy(self):
        L.call("b200dqn_net_comm_destroy", self._h)

    def comm_status(self):
        """-> (mode, healthy): mode 'single' | 'nccl' | 'p2p' (peer-memory exchange); synchronises the device.
        healthy is False when a peer wait timed out since comm_init (results since then are invalid)."""
        mode, err = C.c_int(), C.c_int()
        L.call("b200dqn_net_comm_status", self._h, C.byref(mode), C.byref(err))
        return ("single", "nccl", "p2p")[mode.value], err.value == 0

    @staticmethod
    def comm_unique_id():
        buf = (C.c_char * 128)()
        L.call("b200dqn_comm_unique_id", buf)
        return bytes(buf)

    def launches_per_step(self):
        n = C.c_int()
        L.call("b200dqn_net_launches_per_step", self._h, C.byref(n))
        return n.value
