"""simple_dqn_b200 — the H100-native (sm_90a) replay-and-train hot path behind the call
surface of tambetm/simple_dqn's ReplayMemory / DeepQNetwork / StateBuffer.

Importing the package is cheap; the CUDA library is loaded on first use and there is no CPU
fallback (``_lib.load`` raises if ``libb200dqn.so`` has not been built)."""
from .replay_memory import ReplayMemory, DeviceMinibatch      # noqa: F401
from .state_buffer import StateBuffer, DeviceStates           # noqa: F401
from .deepqnetwork import DeepQNetwork                        # noqa: F401
from ._lib import Stream                                      # noqa: F401

__all__ = ["ReplayMemory", "DeviceMinibatch", "StateBuffer", "DeviceStates", "DeepQNetwork", "Stream"]
