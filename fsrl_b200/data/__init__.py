from .basic_collector import BasicCollector
from .batch import Batch, to_numpy, to_torch_as
from .buffer import DeviceVectorReplayBuffer, ReplayBuffer, VectorReplayBuffer
from .fast_collector import FastCollector
from .traj_buf import TrajectoryBuffer

__all__ = ["Batch", "to_numpy", "to_torch_as", "DeviceVectorReplayBuffer", "VectorReplayBuffer",
           "FastCollector", "ReplayBuffer", "BasicCollector", "TrajectoryBuffer"]
