"""learning/utils/wrappers.py (LW) of the reference, for the batched env and the single-env adapters.

The reference's training and imitation scripts (learning/reinforcement/pytorch/{train,enjoy}_reinforcement.py,
learning/imitation/basic/{train,enjoy}_imitation.py, learning/imitation/tensorflow/train_imitation.py) import their
wrappers from that module and build, innermost first,

    env = launch_env()                # Simulator(640x480, distortion=True, domain_rand=False, ...)
    env = ResizeWrapper(env)          # shape=(120, 160, 3): scipy.misc.imresize, i.e. Pillow's bilinear
    env = NormalizeWrapper(env); env = ImgWrapper(env); env = ActionWrapper(env); env = DtRewardWrapper(env)

With `from gym_duckietown_b200.learning_wrappers import ...` the same lines configure the fused device path: the
frame is rendered at the camera size, resized with Pillow's arithmetic (bit-exact) and written once, already
normalised and transposed, into the observation tensor.  The other classes are the fused ones of `wrappers`.
"""
from __future__ import annotations

from .wrappers import (ActionWrapper, DtRewardWrapper, ImgWrapper, MotionBlurWrapper,  # noqa: F401
                       NormalizeWrapper, _FusedWrapper)

__all__ = ["ResizeWrapper", "NormalizeWrapper", "ImgWrapper", "DtRewardWrapper", "ActionWrapper", "MotionBlurWrapper"]


class ResizeWrapper(_FusedWrapper):
    """LW:39-54 — `scipy.misc.imresize(observation, shape)` on every observation.  For the uint8 RGB frames the env
    emits that is `PIL.Image.fromarray(obs).resize((shape[1], shape[0]), Image.BILINEAR)` (scipy <= 1.2's imresize
    swaps the size to Pillow's (width, height)), a triangle filter widened by the scale factor when it shrinks.
    Here it selects that filter for the env's one device resize slot; the observation space follows the rest of the
    stack, as for the other fused wrappers."""

    def __init__(self, env=None, shape=(120, 160, 3)):
        super().__init__(env)
        shape = tuple(int(s) for s in shape)
        if len(shape) != 3 or shape[2] != 3:
            raise ValueError(f"shape must be (height, width, 3) for the env's RGB frames, not {shape}")
        b = self.batched
        if b.resize is not None:
            raise ValueError(f"the env already resizes its observations to {b.resize[0]}x{b.resize[1]} "
                             f"({b.resize_method}); it has one resize slot, so stacking two resize wrappers would "
                             "drop one")
        self.shape = shape
        b.set_resize(shape[1], shape[0], method="pil_bilinear")
