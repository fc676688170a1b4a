from .rollout_buffer import RolloutBuffer, DeviceRollout, EpisodeRing, FrameRollout  # noqa: F401
from .replay_buffer import ReplayBuffer  # noqa: F401
from .per_buffer import PERBuffer  # noqa: F401
