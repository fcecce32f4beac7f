"""dtsim-b200: batched Duckietown `Simulator.step()` hot path as sm_90a (H100) CUDA kernels.

Public surface (mirrors gym_duckietown's, SURVEY.md 8b):
  Simulator, DuckietownEnv, MultiMapEnv      single-env gym.Env adapters (old 4-tuple API)
  DuckietownLF, DuckietownNav                the lane-following and navigation tasks (envs/duckietown_env.py)
  BatchedDuckietownEnv                       N envs per GPU, torch tensors in/out
  load_map, list_maps                        MapFormat1 loader
  MARKING_NAMES                              names of the lane-marking image's values (markings=True)
  OCCLUSION_NAMES                            names of the occlusion mask's values (flow_occlusion=True)
  BEV_VISIBILITY_NAMES                       names of the bird's-eye visibility's values (bev_visibility=True)
  OBJECT_STATE_NAMES                         names of the object boxes' states (objects=True)
  DONE_CODE_NAMES                            names of the done codes (the state's done_code)
"""
__version__ = "0.1.0"

from .assets import MARKING_NAMES  # noqa: F401
from .lib import BEV_VISIBILITY_NAMES, DONE_CODE_NAMES, OBJECT_STATE_NAMES, OCCLUSION_NAMES  # noqa: F401
from .maps import InvalidMapException, list_maps, load_map  # noqa: F401


def __getattr__(name):  # lazy: importing the package must not require torch/CUDA
    if name in ("BatchedDuckietownEnv", "HostPipeline"):
        from . import batched_env
        return getattr(batched_env, name)
    if name in ("Simulator", "DuckietownEnv", "DuckietownLF", "DuckietownNav", "MultiMapEnv", "NotInLane"):
        from . import simulator
        return getattr(simulator, name)
    raise AttributeError(name)


def _register_envs():
    """One id per map like gym_duckietown/__init__.py:30-46, plus MultiMap-v0."""
    from .gymshim import register
    for _name in list_maps():
        register(id=f"Duckietown-{_name}-v0", entry_point="gym_duckietown_b200.simulator:DuckietownEnv",
                 reward_threshold=400.0, kwargs={"map_name": _name})
    register(id="MultiMap-v0", entry_point="gym_duckietown_b200.simulator:MultiMapEnv", reward_threshold=400.0)


try:
    _register_envs()
except Exception:  # duplicate registration on re-import under real gym
    pass
