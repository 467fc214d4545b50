"""ReplayMemory with the reference's call surface (/root/reference/src/replay_memory.py:6-79),
backed by a ring buffer in HBM and hand-written sm_90a kernels (csrc/replay.cu)."""
import ctypes as C
import logging
import random

import numpy as np

from . import _lib as L

logger = logging.getLogger(__name__)


class _HostMT:
    """Direct view of the MT19937 state inside CPython's process-global generator (``random._inst``), so that the
    per-step lock-step with the host stream costs a few word reads instead of two ``random.getstate()`` calls
    (8 us each: they build a 625-int tuple).  CPython's ``RandomObject`` is ``{PyObject_HEAD; int index;
    uint32_t state[624]}``; the layout is VERIFIED against ``getstate()`` before it is trusted — on any mismatch
    ``probe()`` returns None and the portable getstate()/setstate() path is used."""

    def __init__(self, base, off):
        self._words = (C.c_uint32 * 625).from_address(base + off)      # [0] = index, [1..624] = key
        self.key_ptr = C.c_void_p(base + off + 4)

    @staticmethod
    def probe():
        inst = getattr(random, "_inst", None)
        if inst is None or type(inst).__basicsize__ < 16 + 625 * 4:
            return None
        st = inst.getstate()
        if st[0] != 3 or len(st[1]) != 625:
            return None
        key = st[1]
        raw = (C.c_uint32 * (type(inst).__basicsize__ // 4)).from_address(id(inst))
        for off_words in range(2, len(raw) - 625):
            if raw[off_words] == key[624] and raw[off_words + 1] == key[0] and \
                    list(raw[off_words + 1:off_words + 625]) == list(key[:624]):
                return _HostMT(id(inst), off_words * 4)
        return None

    def pos(self):
        return self._words[0]

    def fingerprint(self):
        w = self._words
        return (w[0], w[1], w[2], w[312], w[624])


_host_mt = False      # False = not probed yet, None = unavailable


def host_mt():
    global _host_mt
    if _host_mt is False:
        try:
            _host_mt = _HostMT.probe()
        except Exception:
            _host_mt = None
    return _host_mt


class DeviceMinibatch(tuple):
    """What ``getMinibatch()`` returns in device mode: a 5-tuple
    ``(prestates, actions, rewards, poststates, terminals)`` like the reference's
    (replay_memory.py:79) whose items are materialised on the host only if somebody looks at
    them (statistics.py:85 does; agent.py:112-114 does not).  ``DeepQNetwork.train`` recognises
    an untouched instance and trains straight from the ring."""

    def __new__(cls, mem, sampled=True):
        self = super().__new__(cls, ())
        self._mem = mem
        self._host = None
        self._ticket = mem._sample_ticket
        self.sampled = sampled       # False: the index draw itself is still pending (it rides in train()'s graph)
        return self

    def _check_current(self):
        assert self._ticket == self._mem._sample_ticket, \
            "this minibatch was overwritten by a later getMinibatch() / set_indexes() / train_fused() before it was used"

    def _materialise(self):
        if self._host is None:
            self._check_current()
            if not self.sampled:
                self._mem._sample_now()
                self.sampled = True
            self._host = self._mem._gather_to_host()
        return self._host

    @property
    def materialised(self):
        return self._host is not None

    def __len__(self):
        return 5

    def __iter__(self):
        return iter(self._materialise())

    def __getitem__(self, i):
        return self._materialise()[i]


class ReplayMemory:
    """rng selects where the index stream of ``random.randint`` (replay_memory.py:59) lives:

    * ``"python"`` (default, exact drop-in): every ``getMinibatch`` uploads ``random.getstate()``,
      samples on the device and writes the advanced state back with ``random.setstate()`` — the
      process-global stream stays in lock-step with what the reference would have consumed.
    * ``"device"``: the MT19937 state is taken from ``random.getstate()`` once and then lives on
      the GPU (no host round trip per step; the host ``random`` is not advanced).

    device_minibatch=True makes ``getMinibatch`` return a :class:`DeviceMinibatch`.
    """

    def __init__(self, size, args, device=0, rng="python", device_minibatch=False, stream=None):
        self.size = int(size)
        self.history_length = args.history_length
        self.dims = (args.screen_height, args.screen_width)
        self.batch_size = args.batch_size
        self.device = device
        self.rng_mode = rng
        self.device_minibatch = device_minibatch
        self._stream_obj = stream            # keep the stream alive as long as this object uses it
        self._stream = L.stream_ptr(stream)
        assert rng in ("python", "device")
        h = C.c_void_p()
        L.call("b200dqn_replay_create", device, self.size, self.dims[0], self.dims[1], self.history_length,
               self.batch_size, C.byref(h))
        self._h = h
        # pre-allocated host minibatch buffers, returned by reference like the original's (:21-22, :79)
        self.prestates = np.empty((self.batch_size, self.history_length) + self.dims, dtype=np.uint8)
        self.poststates = np.empty((self.batch_size, self.history_length) + self.dims, dtype=np.uint8)
        self._rng_on_device = False
        self._host_state_in_sync = None       # host `random` state (or its fingerprint) known to equal the device stream
        self._mt = host_mt() if rng == "python" else None
        self._sample_ticket = 0
        self.last_indexes = None
        self.last_words_consumed = None
        logger.info("Replay memory size: %d" % self.size)
        # proportional prioritized replay (Schaul et al., 2016), parameters named as in OpenAI baselines: a new
        # capability, off unless args.prioritized_replay is set.  beta is annealed to 1 over beta_steps samplings,
        # by default the number of train steps the reference's main loop runs.
        self.prioritized = False
        self.alpha = getattr(args, "alpha", 0.6)
        self.beta0 = getattr(args, "beta0", 0.4)
        self.eps = getattr(args, "eps", 1e-6)
        self.beta_steps = getattr(args, "beta_steps", None)
        if self.beta_steps is None:
            self.beta_steps = (getattr(args, "epochs", 200) * getattr(args, "train_steps", 250000) //
                               getattr(args, "train_frequency", 4) * getattr(args, "train_repeat", 1))
        if getattr(args, "prioritized_replay", False):
            self.set_prioritized(True)
        # n-step returns (Hessel et al., 2018): a new capability, one-step (the reference) unless args.n_step > 1
        self.n_step = 1
        if getattr(args, "n_step", 1) != 1:
            self.set_n_step(args.n_step)

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            try:
                L.load().b200dqn_replay_destroy(h)
            except Exception:
                pass

    # ---- cursor attributes of the reference (:17-18)
    def _cursor(self):
        c, cur = C.c_int64(), C.c_int64()
        L.call("b200dqn_replay_get_cursor", self._h, C.byref(c), C.byref(cur))
        return c.value, cur.value

    @property
    def count(self):
        return self._cursor()[0]

    @property
    def current(self):
        return self._cursor()[1]

    def set_cursor(self, count, current):
        L.call("b200dqn_replay_set_cursor", self._h, int(count), int(current))

    # ---- ring arrays of the reference (:10-13) as on-demand host copies
    def _download(self, which, dtype, shape):
        view = self.device_view(which, dtype, shape)
        return L.download(self.device, view.ptr, shape, dtype, self._stream)

    def device_view(self, which, dtype, shape):
        p, b = C.c_void_p(), C.c_size_t()
        L.call("b200dqn_replay_device_ptr", self._h, which, C.byref(p), C.byref(b))
        return L.DeviceArray(p.value, shape, np.dtype(dtype).str, owner=self)

    @property
    def actions(self):
        return self._download(L.PTR_ACTIONS, np.uint8, (self.size,))

    @property
    def rewards(self):
        return self._download(L.PTR_REWARDS, np.int64, (self.size,))

    @property
    def terminals(self):
        return self._download(L.PTR_TERMINALS, np.uint8, (self.size,)).astype(np.bool_)

    @property
    def screens(self):
        return self._download(L.PTR_SCREENS, np.uint8, (self.size,) + self.dims)

    # ---- prioritized replay
    def set_prioritized(self, on=True, alpha=None, beta0=None, beta_steps=None, eps=None):
        """Switch proportional prioritized replay on or off (include/b200dqn.h, b200dqn_replay_set_prioritized).
        Switching on resets every stored priority and max_priority to 1.  Parameters left None keep their values."""
        self.alpha = self.alpha if alpha is None else alpha
        self.beta0 = self.beta0 if beta0 is None else beta0
        self.beta_steps = self.beta_steps if beta_steps is None else beta_steps
        self.eps = self.eps if eps is None else eps
        L.call("b200dqn_replay_set_prioritized", self._h, int(bool(on)), float(self.alpha), float(self.beta0),
               float(self.beta_steps), float(self.eps))
        self.prioritized = bool(on)

    @property
    def priorities(self):
        """Host copy of the stored priorities p^alpha, float64 (size,)."""
        assert self.prioritized or self._has_per_buffers(), "prioritized replay was never switched on"
        return self._download(L.PTR_PRIORITIES, np.float64, (self.size,))

    @property
    def last_weights(self):
        """Importance weights of the last prioritized draw (or set_indexes), float32 (batch,)."""
        assert self.prioritized or self._has_per_buffers(), "prioritized replay was never switched on"
        return self._download(L.PTR_IS_WEIGHTS, np.float32, (self.batch_size,))

    @property
    def max_priority(self):
        return float(self._download(L.PTR_MAX_PRIORITY, np.float64, (1,))[0])

    def _has_per_buffers(self):
        p, b = C.c_void_p(), C.c_size_t()
        L.call("b200dqn_replay_device_ptr", self._h, L.PTR_PRIORITIES, C.byref(p), C.byref(b))
        return b.value > 0

    # ---- n-step returns
    def set_n_step(self, n):
        """Train on n-step returns (include/b200dqn.h, b200dqn_replay_set_n_step): a sample's poststate is
        getState(index + n - 1) and its target sums the discounted rewards of index .. index + n - 1, cut at the first
        terminal.  n = 1 is the reference's step.  Raises AssertionError unless 1 <= n and history_length + n <= size.
        A minibatch handed out before the switch can no longer be trained."""
        L.call("b200dqn_replay_set_n_step", self._h, int(n))
        self.n_step = int(n)
        self._sample_ticket += 1

    # ---- reference methods
    def add(self, action, reward, screen, terminal):
        assert screen.shape == self.dims                               # :27
        if screen.dtype != np.uint8 or not screen.flags["C_CONTIGUOUS"]:
            screen = np.ascontiguousarray(screen, dtype=np.uint8)
        # rewards is an int64 array (:11): a float reward is truncated toward zero on store, as numpy does
        L.call("b200dqn_replay_add", self._h, int(action), int(reward), screen.ctypes.data, 1 if terminal else 0,
               self._stream)

    def add_batch(self, actions, rewards, screens, terminals):
        """n consecutive add() calls in one transfer."""
        n = len(actions)
        assert screens.shape == (n,) + self.dims
        a = np.ascontiguousarray(actions, dtype=np.uint8)
        r = np.ascontiguousarray(rewards, dtype=np.int64)
        s = np.ascontiguousarray(screens, dtype=np.uint8)
        t = np.ascontiguousarray(terminals, dtype=np.uint8)
        L.call("b200dqn_replay_add_batch", self._h, n, L.np_ptr(a), L.np_ptr(r), L.np_ptr(s), L.np_ptr(t),
               self._stream)

    def getState(self, index):
        out = np.empty((self.history_length,) + self.dims, dtype=np.uint8)
        try:
            L.call("b200dqn_replay_get_state", self._h, int(index), L.np_ptr(out), self._stream)
        except L.B200DQNError as e:
            if e.code == L.ESTATE:
                raise AssertionError(str(e))                          # :38
            raise
        return out

    # ---- sampling
    def seed_device_rng(self, rnd=random):
        """Adopt the MT19937 state of ``rnd`` (default: the process-global ``random``)."""
        st = rnd.getstate()
        assert st[0] == 3
        key = np.array(st[1], dtype=np.uint32)
        L.call("b200dqn_replay_set_rng", self._h, L.np_ptr(key), self._stream)
        self._rng_on_device = True
        self._host_state_in_sync = None       # the device stream no longer (provably) equals the global one

    def read_device_rng(self):
        key = np.empty(625, dtype=np.uint32)
        L.call("b200dqn_replay_get_rng", self._h, L.np_ptr(key), self._stream)
        return key

    # ---- lock-step with the process-global `random` (rng="python")
    def _host_upload_args(self):
        """(key pointer or None, position): what the device must adopt before its next draw — None when the host
        stream has not moved since the device last matched it."""
        mt = self._mt
        if mt is not None:
            if mt.fingerprint() == self._host_state_in_sync:
                return None, 0
            return mt.key_ptr, mt.pos()
        st = random.getstate()[1]
        if st == self._host_state_in_sync:
            return None, 0
        self._key_keepalive = np.array(st, dtype=np.uint32)
        return L.np_ptr(self._key_keepalive), int(st[624])

    def _host_advance(self, words):
        """The device consumed `words` 32-bit outputs (one per trial of replay_memory.py:59): so does the host."""
        grb = random.getrandbits
        for _ in range(words):
            grb(32)
        self._host_state_in_sync = self._mt.fingerprint() if self._mt is not None else random.getstate()[1]
        self._rng_on_device = True
        self.last_words_consumed = words

    def _sample_now(self):
        if self.rng_mode == "python":
            key, pos = self._host_upload_args()
            if key is not None:
                L.call("b200dqn_replay_set_rng_parts", self._h, key, pos, self._stream)
            words = C.c_uint32()
            L.call("b200dqn_replay_sample_sync", self._h, C.byref(words), self._stream)
            self._host_advance(words.value)
        else:
            if not self._rng_on_device:
                self.seed_device_rng(random)
            L.call("b200dqn_replay_sample", self._h, self._stream)

    def sample(self):
        """The index draw of getMinibatch (:55-69) on the device.  rng="python": in lock-step with the process-global
        stream — its state is uploaded only if somebody else drew from `random` since our last sample, and the host
        is advanced by exactly the number of 32-bit words the device consumed."""
        assert self.count >= self.history_length + self.n_step         # :52 at n_step 1
        self._sample_now()
        self._sample_ticket += 1

    def set_indexes(self, indexes):
        idx = np.ascontiguousarray(indexes, dtype=np.int32)
        assert idx.shape == (self.batch_size,)
        L.call("b200dqn_replay_set_indexes", self._h, L.np_ptr(idx), self._stream)
        self._sample_ticket += 1

    def _gather_to_host(self):
        """The reference's 5-tuple; with n_step > 1 rewards and terminals are (batch, n_step) windows starting at the
        index, and the poststates are getState(index + n_step - 1)."""
        L.call("b200dqn_replay_gather", self._h, self._stream)
        mb = (self.batch_size,) if self.n_step == 1 else (self.batch_size, self.n_step)
        actions = np.empty(self.batch_size, dtype=np.uint8)
        rewards = np.empty(mb, dtype=np.int64)
        terminals = np.empty(mb, dtype=np.uint8)
        indexes = np.empty(self.batch_size, dtype=np.int32)
        words = np.zeros(1, dtype=np.uint32)
        L.call("b200dqn_replay_read_minibatch", self._h, L.np_ptr(self.prestates), L.np_ptr(actions),
               L.np_ptr(rewards), L.np_ptr(self.poststates), L.np_ptr(terminals), L.np_ptr(indexes),
               L.np_ptr(words), self._stream)
        self.last_indexes = indexes
        self.last_words_consumed = int(words[0])
        return self.prestates, actions, rewards, self.poststates, terminals.astype(np.bool_)

    def getMinibatch(self):
        # replay_memory.py:50-79
        # a prioritized or n-step minibatch must train from the ring
        if self.device_minibatch or self.prioritized or self.n_step > 1:
            # agent.py:112-114 is `mb = mem.getMinibatch(); net.train(mb, epoch)` with nothing in between: hand out
            # a handle and let the draw ride in train()'s graph (one launch, one wait per step).  Anything else that
            # looks at the handle (statistics.py:85) triggers the draw on the spot.
            assert self.count >= self.history_length + self.n_step     # :52 at n_step 1
            self._sample_ticket += 1
            return DeviceMinibatch(self, sampled=False)
        self.sample()
        return self._gather_to_host()
