"""ctypes binding of libb200dqn.so (include/b200dqn.h).  There is NO fallback: if the CUDA
library is missing or a call fails, this raises — the product never computes on the CPU."""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libb200dqn.so")

OK, EINVAL, ECUDA, ENOTIMPL, ENCCL, ESTATE = 0, -1, -2, -3, -4, -5
MATH_FP32_SIMT, MATH_TCGEN05 = 0, 1
OPT_RMSPROP, OPT_ADAM, OPT_ADADELTA = 0, 1, 2

(PTR_SCREENS, PTR_ACTIONS, PTR_REWARDS, PTR_TERMINALS, PTR_PRESTATES, PTR_POSTSTATES, PTR_MB_ACTIONS,
 PTR_MB_REWARDS, PTR_MB_TERMINALS, PTR_INDEXES, PTR_WORDS_CONSUMED, PTR_MT_STATE, PTR_PRIORITIES, PTR_SUM_TREE,
 PTR_IS_WEIGHTS, PTR_MAX_PRIORITY, PTR_MIN_TREE) = range(17)
(NET_PTR_Q_ONLINE, NET_PTR_Q_TARGET, NET_PTR_DELTAS, NET_PTR_GRADS, NET_PTR_WEIGHTS, NET_PTR_COST, NET_PTR_H1,
 NET_PTR_H2, NET_PTR_H3, NET_PTR_H4, NET_PTR_DZ4, NET_PTR_DZ3, NET_PTR_DZ2, NET_PTR_DZ1,
 NET_PTR_Q_ONLINE_POST, NET_PTR_TD_ERRORS, NET_PTR_ROW_COSTS, NET_PTR_LOGITS, NET_PTR_PROBS, NET_PTR_TARGET_DIST,
 NET_PTR_LOGIT_GRADS, NET_PTR_DZ4_PLANES, NET_PTR_DUELING_VA, NET_PTR_QUANTILES, NET_PTR_TARGET_QUANTILES,
 NET_PTR_QUANTILE_GRADS, NET_PTR_Q_TARGET_PRE, NET_PTR_TD_TARGETS, NET_PTR_IQN_TAUS, NET_PTR_IQN_COS, NET_PTR_IQN_PHI,
 NET_PTR_IQN_X, NET_PTR_IQN_QUANTILES, NET_PTR_IQN_TARGET_QUANTILES, NET_PTR_IQN_QUANTILE_GRADS, NET_PTR_IQN_DX,
 NET_PTR_IQN_DPHI, NET_PTR_IQN_TAU_COUNTER, NET_PTR_SHIFT_OFFSETS, NET_PTR_SHIFT_DRAWS, NET_PTR_REM_HEADS,
 NET_PTR_REM_ALPHAS, NET_PTR_REM_GRADS, NET_PTR_REM_COUNTER, NET_PTR_FQF_LOGITS, NET_PTR_FQF_PROBS,
 NET_PTR_FQF_FRACTIONS, NET_PTR_FQF_BOUNDARY_QUANTILES, NET_PTR_FQF_FRACTION_GRADS, NET_PTR_FQF_LOGIT_GRADS,
 NET_PTR_BOOT_MASKS, NET_PTR_BOOT_TARGETS, NET_PTR_BOOT_DELTAS, NET_PTR_BOOT_ACTIVE_HEAD, NET_PTR_GRAD_SQ,
 NET_PTR_GRAD_NORM, NET_PTR_CLIP_SCALE) = range(57)


class B200DQNError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("libb200dqn error %d: %s" % (code, msg))
        self.code = code


class NetConfig(C.Structure):
    _fields_ = [("num_actions", C.c_int), ("batch_size", C.c_int), ("history_length", C.c_int),
                ("screen_h", C.c_int), ("screen_w", C.c_int), ("discount_rate", C.c_double),
                ("learning_rate", C.c_double), ("decay_rate", C.c_double), ("clip_error", C.c_double),
                ("min_reward", C.c_double), ("max_reward", C.c_double), ("target_steps", C.c_int),
                ("math_mode", C.c_int), ("optimizer", C.c_int), ("num_atoms", C.c_int), ("v_min", C.c_double),
                ("v_max", C.c_double), ("dueling", C.c_int), ("num_quantiles", C.c_int),
                ("munchausen", C.c_int), ("munchausen_alpha", C.c_double), ("munchausen_tau", C.c_double),
                ("munchausen_clip", C.c_double), ("num_tau_samples", C.c_int), ("num_quantile_samples", C.c_int),
                ("tau_seed", C.c_uint64), ("random_shift", C.c_int), ("shift_seed", C.c_uint64),
                ("num_heads", C.c_int), ("rem_seed", C.c_uint64),
                ("num_fractions", C.c_int), ("fraction_lr", C.c_double),
                ("bootstrap_heads", C.c_int), ("bootstrap_p", C.c_double), ("bootstrap_seed", C.c_uint64),
                ("soft_target_tau", C.c_double), ("max_grad_norm", C.c_double)]


_P = C.c_void_p
_u8p = C.POINTER(C.c_uint8)
_i32p = C.POINTER(C.c_int32)
_i64p = C.POINTER(C.c_int64)
_u32p = C.POINTER(C.c_uint32)
_f32p = C.POINTER(C.c_float)

# name -> argtypes; every function returns int status except the two noted below
SIGNATURES = {
    "b200dqn_device_info": [C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int),
                            C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)],
    "b200dqn_copy_to_host": [C.c_int, _P, _P, C.c_size_t, _P],
    "b200dqn_copy_to_device": [C.c_int, _P, _P, C.c_size_t, _P],
    "b200dqn_stream_create": [C.c_int, C.POINTER(_P)],
    "b200dqn_stream_destroy": [C.c_int, _P],
    "b200dqn_stream_synchronize": [C.c_int, _P],
    "b200dqn_ktrace_begin": [C.c_int],
    "b200dqn_ktrace_begin_at": [C.c_int, C.c_int],
    "b200dqn_ktrace_end": [C.c_int, _P, _P, _P, C.POINTER(C.c_int)],
    "b200dqn_profile_begin": [C.c_int, _P],
    "b200dqn_profile_end": [C.c_int, _P, _P, C.POINTER(C.c_int)],
    "b200dqn_replay_create": [C.c_int, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(_P)],
    "b200dqn_replay_destroy": [_P],
    "b200dqn_replay_add": [_P, C.c_int, C.c_int64, _P, C.c_int, _P],
    "b200dqn_replay_add_batch": [_P, C.c_int64, _P, _P, _P, _P, _P],
    "b200dqn_replay_get_cursor": [_P, _i64p, _i64p],
    "b200dqn_replay_set_cursor": [_P, C.c_int64, C.c_int64],
    "b200dqn_replay_get_state": [_P, C.c_int64, _P, _P],
    "b200dqn_replay_set_rng": [_P, _P, _P],
    "b200dqn_replay_get_rng": [_P, _P, _P],
    "b200dqn_replay_set_rng_parts": [_P, _P, C.c_uint32, _P],
    "b200dqn_replay_sample": [_P, _P],
    "b200dqn_replay_sample_sync": [_P, _u32p, _P],
    "b200dqn_replay_set_indexes": [_P, _P, _P],
    "b200dqn_replay_gather": [_P, _P],
    "b200dqn_replay_read_minibatch": [_P, _P, _P, _P, _P, _P, _P, _P, _P],
    "b200dqn_replay_device_ptr": [_P, C.c_int, C.POINTER(_P), C.POINTER(C.c_size_t)],
    "b200dqn_replay_set_prioritized": [_P, C.c_int, C.c_double, C.c_double, C.c_double, C.c_double],
    "b200dqn_replay_set_n_step": [_P, C.c_int],
    "b200dqn_statebuf_create": [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(_P)],
    "b200dqn_statebuf_destroy": [_P],
    "b200dqn_statebuf_add": [_P, _P, _P],
    "b200dqn_statebuf_reset": [_P, _P],
    "b200dqn_statebuf_read": [_P, _P, C.c_int, _P],
    "b200dqn_statebuf_device_ptr": [_P, C.POINTER(_P), C.POINTER(C.c_size_t)],
    "b200dqn_net_config_default": [C.POINTER(NetConfig), C.c_int],
    "b200dqn_net_create": [C.c_int, C.POINTER(NetConfig), C.POINTER(_P)],
    "b200dqn_net_destroy": [_P],
    "b200dqn_net_set_weights": [_P, C.c_int, C.c_int, _P, _P, _P],
    "b200dqn_net_get_weights": [_P, C.c_int, C.c_int, _P, _P, _P],
    "b200dqn_net_layer_shape": [_P, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)],
    "b200dqn_net_num_states": [_P, C.POINTER(C.c_int)],
    "b200dqn_net_set_state": [_P, C.c_int, C.c_int, C.c_int, _P, _P],
    "b200dqn_net_get_state": [_P, C.c_int, C.c_int, C.c_int, _P, _P],
    "b200dqn_net_sync_target": [_P, _P],
    "b200dqn_net_soft_update_target": [_P, C.c_double, _P],
    "b200dqn_net_predict": [_P, _P, _P, _P],
    "b200dqn_net_predict_device": [_P, _P, C.c_int, _P, _P],
    "b200dqn_net_predict_device_host": [_P, _P, C.c_int, _P, _P],
    "b200dqn_net_train": [_P, _P, _P, _P, _P, _P, _f32p, _P],
    "b200dqn_net_train_device": [_P, _P, _P, _P, _P, _P, _P],
    "b200dqn_net_train_sampled": [_P, _P, _P],
    "b200dqn_net_train_sampled_cost": [_P, _P, _f32p, _P],
    "b200dqn_net_train_fused": [_P, _P, C.c_int, _P],
    "b200dqn_net_step_host": [_P, _P, C.c_int, _P, _P, _P, _P, C.c_int, _P, C.c_uint32, _P, _P, _P],
    "b200dqn_net_read_costs": [_P, C.c_int, _P, _P],
    "b200dqn_net_train_iterations": [_P, _i64p],
    "b200dqn_net_device_ptr": [_P, C.c_int, C.POINTER(_P), C.POINTER(C.c_size_t)],
    "b200dqn_net_set_keep_grads": [_P, C.c_int],
    "b200dqn_net_set_double_q": [_P, C.c_int],
    "b200dqn_net_set_active_head": [_P, C.c_int, _P],
    "b200dqn_net_get_grads": [_P, C.c_int, _P, _P],
    "b200dqn_net_launches_per_step": [_P, C.POINTER(C.c_int)],
    "b200dqn_debug_trace": [_P, C.c_int],
    "b200dqn_comm_unique_id": [_P],
    "b200dqn_net_comm_init": [_P, _P, C.c_int, C.c_int],
    "b200dqn_net_comm_destroy": [_P],
    "b200dqn_net_comm_status": [_P, _P, _P],
    "b200dqn_debug_xchg": [_P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P, _P],
}
EXPORTS = sorted(list(SIGNATURES) + ["b200dqn_last_error", "b200dqn_version"])

_lib = None


def load():
    """Return the loaded library, loading it on first use.  Raises if it is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            "simple_dqn_b200: %s is missing — build it with `python -m simple_dqn_b200.build` "
            "(nvcc, sm_90a).  There is no CPU fallback." % LIB_PATH)
    lib = C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)
    lib.b200dqn_last_error.restype = C.c_char_p
    lib.b200dqn_last_error.argtypes = []
    lib.b200dqn_version.restype = C.c_int
    lib.b200dqn_version.argtypes = []
    for name, args in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.argtypes = args
        fn.restype = C.c_int
    _lib = lib
    return lib


def debug_trace(n=96):
    import numpy as np
    out = np.zeros(n, dtype=np.uint64)
    got = load().b200dqn_debug_trace(np_ptr(out), n)
    return out[:max(got, 0)]


def check(rc):
    if rc != OK:
        msg = load().b200dqn_last_error().decode("utf-8", "replace")
        if rc == ENOTIMPL:
            raise NotImplementedError(msg)
        if rc == EINVAL:
            raise AssertionError(msg)        # the reference's error convention is `assert`
        raise B200DQNError(rc, msg)


def call(name, *args):
    check(getattr(load(), name)(*args))


def np_ptr(a):
    """void* of a C-contiguous numpy array (or None)."""
    if a is None:
        return None
    assert a.flags["C_CONTIGUOUS"], "array must be C-contiguous"
    return a.ctypes.data_as(C.c_void_p)


def stream_ptr(stream):
    """Accept None, an int handle, or an object with .cuda_stream (torch.cuda.Stream)."""
    if stream is None:
        return None
    if hasattr(stream, "cuda_stream"):
        return C.c_void_p(stream.cuda_stream)
    return C.c_void_p(int(stream))


class DeviceArray:
    """Zero-copy view of library-owned device memory: exposes __cuda_array_interface__ so
    ``torch.as_tensor(view, device='cuda')`` / cupy can wrap it without a copy."""

    def __init__(self, ptr, shape, typestr, owner=None):
        self.ptr = int(ptr)
        self.shape = tuple(int(s) for s in shape)
        self.typestr = typestr
        self._owner = owner            # keeps the owning object alive
        self.__cuda_array_interface__ = {"shape": self.shape, "typestr": typestr, "data": (self.ptr, False),
                                         "version": 2, "strides": None}


def download(device, dev_ptr, shape, dtype, stream=None):
    """Host numpy copy of a library-owned device buffer."""
    import numpy as np
    out = np.empty(shape, dtype=dtype)
    call("b200dqn_copy_to_host", device, np_ptr(out), C.c_void_p(int(dev_ptr)), out.nbytes, stream)
    return out


def profile_begin(device=0, stream=None):
    call("b200dqn_profile_begin", device, stream)


def profile_end(max_entries=8192):
    """[(label, ms), ...] for every kernel launched since profile_begin, in launch order."""
    import numpy as np
    names = C.create_string_buffer(max_entries * 32)
    ms = np.zeros(max_entries, dtype=np.float32)
    n = C.c_int()
    call("b200dqn_profile_end", max_entries, names, np_ptr(ms), C.byref(n))
    raw = names.raw
    return [(raw[i * 32:(i + 1) * 32].split(b"\0")[0].decode(), float(ms[i])) for i in range(n.value)]


class Stream:
    """A library-owned non-blocking CUDA stream (``.cuda_stream`` like torch.cuda.Stream)."""

    def __init__(self, device=0):
        h = C.c_void_p()
        call("b200dqn_stream_create", device, C.byref(h))
        self.device = device
        self.cuda_stream = h.value

    def synchronize(self):
        call("b200dqn_stream_synchronize", self.device, C.c_void_p(self.cuda_stream))

    def __del__(self):
        h, self.cuda_stream = getattr(self, "cuda_stream", None), None
        if h:
            try:
                load().b200dqn_stream_destroy(self.device, C.c_void_p(h))
            except Exception:
                pass


def ktrace_begin(device=0, step=0):
    """Arm the in-graph timeline; step >= 1 records only that fused step after arming (steady state)."""
    call("b200dqn_ktrace_begin_at", device, step)


def ktrace_end(max_entries=128):
    """[(label, start_ns, end_ns)] of every instrumented launch since ktrace_begin (GPU globaltimer)."""
    import numpy as np
    names = C.create_string_buffer(max_entries * 32)
    st = np.zeros(max_entries, dtype=np.uint64)
    en = np.zeros(max_entries, dtype=np.uint64)
    n = C.c_int()
    call("b200dqn_ktrace_end", max_entries, names, np_ptr(st), np_ptr(en), C.byref(n))
    raw = names.raw
    return [(raw[i * 32:(i + 1) * 32].split(b"\0")[0].decode(), int(st[i]), int(en[i])) for i in range(n.value)]
