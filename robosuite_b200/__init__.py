"""H100-native batched manipulation simulator keeping robosuite's make / reset / step / controller_config surface."""
import os as _os

__version__ = "0.2.0"

# The engine replays one CUDA graph per environment group on its own stream (8+ streams per task handle).  A process has 8 hardware
# work queues by default; streams beyond the eighth share a queue and falsely serialise.  Honoured only if CUDA is not initialised
# yet - import robosuite_b200 before the first CUDA call, or export the variable yourself.
_os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")


def make(env_name, *args, **kwargs):
    from .envs import make as _make

    return _make(env_name, *args, **kwargs)
