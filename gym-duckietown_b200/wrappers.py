"""The reference's wrapper classes for the BATCHED env, as configuration of the fused device path.

In gym-duckietown a wrapper is a Python object that post-processes one env's numpy observation / reward / action
per step (src/gym_duckietown/wrappers.py = W, learning/utils/wrappers.py = LW).  On a batch of thousands of envs
each such pass would re-read and re-write the whole observation batch (236 MB per step at 4096 x 160x120), so here
the same classes only *select* what the step kernels emit (`dts_set_output_format`): layout and dtype are applied
by the rasteriser's resolve, the reward map and the action decoding by the per-env logic kernel.  Same names,
same constructor arguments, same resulting observation_space as the reference classes:

    env = BatchedDuckietownEnv(4096, "small_loop", camera_width=160, camera_height=120, ...)
    env = DtRewardWrapper(ActionWrapper(ImgWrapper(NormalizeWrapper(env))))      # LW training stack
    obs, reward, done, info = env.step(actions)      # obs f32[N,3,H,W] in [0,1], written once by the GPU

`ResizeWrapper` runs cv2.INTER_CUBIC's 8-bit arithmetic in a device pass right after the render
(`dts_set_resize`), so the resized batch — not the full frames — is what a host-facing pipeline copies out.
`UndistortWrapper`'s rectification is a second table of the render's fused gather (`dts_set_rectify_lut`): the
rectified frame is rendered directly, with no extra pass.
"""
from __future__ import annotations

import numpy as np

from .gymshim import spaces


class _FusedWrapper:
    """Forwards everything to the wrapped batched env; subclasses flip one switch of its output format."""

    def __init__(self, env):
        self.env = env

    @property
    def batched(self):
        """The BatchedDuckietownEnv whose device path the wrapper configures: the wrapped env itself, or the one inside
        a single-env adapter (simulator.Simulator / DuckietownEnv keep it as `_b`)."""
        e = self.env
        while not hasattr(e, "set_output_format"):
            e = e._b if hasattr(e, "_b") else e.env
        return e

    def __getattr__(self, name):
        if name == "env":
            raise AttributeError(name)
        return getattr(self.env, name)

    @property
    def unwrapped(self):
        return getattr(self.env, "unwrapped", self.env)

    @property
    def observation_space(self):
        b = self.batched
        f = b.output_format
        H, W = b.obs_size
        shape = {"hwc": (H, W, 3), "chw": (3, H, W), "cwh": (3, W, H)}[f["obs_layout"]]
        if f["obs_dtype"] == "float32":
            return spaces.Box(0.0, 1.0, shape, dtype=np.float32)
        return spaces.Box(0, 255, shape, dtype=np.uint8)

    def step(self, actions, **kw):
        return self.env.step(actions, **kw)

    def reset(self, *a, **kw):
        return self.env.reset(*a, **kw)

    def _wrapped(self):
        """The fused wrappers below this one, outermost first."""
        e = self.env
        while isinstance(e, _FusedWrapper):
            yield e
            e = e.env


class ImgWrapper(_FusedWrapper):
    """LW:73-87 — HWC -> CHW."""

    def __init__(self, env=None):
        super().__init__(env)
        self.batched.set_output_format(obs_layout="chw")


class PyTorchObsWrapper(_FusedWrapper):
    """W:93-110 — `transpose(2, 1, 0)`: HWC -> C x W x H (sic)."""

    def __init__(self, env=None):
        super().__init__(env)
        self.batched.set_output_format(obs_layout="cwh")


class NormalizeWrapper(_FusedWrapper):
    """LW:56-70 — (obs - low) / (high - low) with low = 0, high = 255, as float32."""

    def __init__(self, env=None):
        super().__init__(env)
        self.batched.set_output_format(obs_dtype="float32")


class DtRewardWrapper(_FusedWrapper):
    """LW:90-102 — -1000 -> -10, positive rewards + 10, the rest + 4."""

    def __init__(self, env):
        super().__init__(env)
        self.batched.set_output_format(reward="dt")


class ActionWrapper(_FusedWrapper):
    """LW:106-112 — velocity command scaled by 0.8 ("at max speed the duckie can't turn anymore")."""

    def __init__(self, env):
        super().__init__(env)
        self.batched.set_output_format(action_vel_scale=0.8)


class DiscreteWrapper(_FusedWrapper):
    """W:8-33 — three actions (0 left, 1 right, 2 forward); pass the ids as int / float tensor of shape [N]."""

    def __init__(self, env):
        super().__init__(env)
        self.batched.set_output_format(discrete_actions=True)
        self.action_space = spaces.Discrete(3)

    def step(self, actions, **kw):
        import torch
        b = self.batched
        ids = actions.to(device=b.device, dtype=torch.float32).reshape(b.num_envs)
        return self.env.step(torch.stack([ids, torch.zeros_like(ids)], dim=1), **kw)


class SteeringToWheelVelWrapper(_FusedWrapper):
    """W:36-90 — [vel, steering] -> wheel duty.  The batched env does this conversion itself when built with
    action_mode='vel_steer' (DuckietownEnv.step); wrapping a 'pwm' env is therefore a configuration error."""

    def __init__(self, env, gain=1.0, trim=0.0, radius=0.0318, k=27.0, limit=1.0):
        super().__init__(env)
        c = self.batched.cfg
        if c.action_mode != 1:
            raise ValueError("build the env with action_mode='vel_steer' and these gain/trim/radius/k/limit instead")
        if (c.gain, c.trim, c.radius, c.k, c.limit) != (gain, trim, radius, k, limit):
            raise ValueError("wrapper parameters differ from the env's: pass them to BatchedDuckietownEnv(gain=..., ...)")


class ResizeWrapper(_FusedWrapper):
    """W:111-141 — `cv2.resize(obs.swapaxes(0, 2), dsize=(resize_w, resize_h), interpolation=cv2.INTER_CUBIC).swapaxes(0, 2)`
    on reset and step.  The reference applies it on top of PyTorchObsWrapper ([C, W, H] observations, hence the
    swapaxes); here it is a switch of the device path like the others: the env then emits resize_h x resize_w frames in
    whatever layout / dtype the rest of the stack selected."""

    def __init__(self, env=None, resize_w=80, resize_h=80):
        super().__init__(env)
        self.resize_w, self.resize_h = resize_w, resize_h
        self.batched.set_resize(resize_w, resize_h)


class UndistortWrapper(_FusedWrapper):
    """W:145-227 — the env renders without its fisheye (`unwrapped.undistort = True`) and every reset / step observation
    is `cv2.remap(obs, mapx, mapy, cv2.INTER_NEAREST)` with the map `cv2.initUndistortRectifyMap(K, D, I, P, (W, H),
    CV_32FC1)` at the observation's size (distortion.rectify_maps).  Here that gather runs inside the render through a
    second table of the fused fisheye kernels (BatchedDuckietownEnv.set_rectification): the rectified frame is rendered
    directly.  `render_obs()` stays the pinhole frame, as in the reference.

    Stacking: resize, layout and dtype wrappers may go above this one (the resize pass reads the rectified render; a
    nearest gather commutes with /255 and with the transposes).  Below it they are refused — the reference would then
    build the map at the resized or transposed shape — and so is MotionBlurWrapper in either order."""

    def __init__(self, env=None):
        super().__init__(env)
        assert self.unwrapped.distortion, "Distortion is false, no need for this wrapper"
        b = self.batched
        if b.resize is not None:
            raise ValueError(f"the env already resizes its observations to {b.resize[0]}x{b.resize[1]}: put "
                             "UndistortWrapper below the resize wrapper, whose pass then reads the rectified frames")
        if b.output_format["obs_layout"] != "hwc":
            raise ValueError(f"the env emits {b.output_format['obs_layout'].upper()} observations: put UndistortWrapper "
                             "below the layout wrapper, so that its map is built for H x W x 3 frames")
        if any(isinstance(w, MotionBlurWrapper) for w in self._wrapped()):
            raise ValueError("UndistortWrapper does not go on top of MotionBlurWrapper")
        from .distortion import rectify_maps
        self.mapx, self.mapy = rectify_maps(b.camera_width, b.camera_height)
        b.set_rectification(self.mapx, self.mapy)
        self.unwrapped.undistort = True                                      # W:159


class MotionBlurWrapper(_FusedWrapper):
    """LW:8-54 — the reference class sets `frame_skip = 3`, divides the wrapped env's delta_time by it and, per step,
    renders before each of three `update_physics(action)` calls and once after, returning
    `np.average(window, axis=0, weights=[0.8, 0.15, 0.04, 0.01])` (float64, oldest frame heaviest) with the reward /
    done of the final state.  `action` is what update_physics takes: wheel commands, clipped to [-1, 1].
    Here: three physics-only device steps with a render in between, then one blend kernel (dts_blend4)."""

    WEIGHTS = (0.8, 0.15, 0.04, 0.01)

    def __init__(self, env=None):
        super().__init__(env)
        import torch
        b = self.batched
        if b.auto_reset:
            raise ValueError("MotionBlurWrapper steps the physics three times per step: build the env without auto_reset")
        if b.undistort:
            raise ValueError("MotionBlurWrapper does not go on top of UndistortWrapper or an env with undistort set")
        self.frame_skip = 3
        b.delta_time = b.delta_time / self.frame_skip                       # LW:14
        from . import lib as L
        b.sim.set_timing(b.delta_time, 1, L.ACTION_PWM)                     # update_physics(action): one physics step per call
        with torch.cuda.device(b.device):
            self._window = [torch.empty_like(b.obs) for _ in range(4)]
            self._blurred = torch.empty(tuple(b.obs.shape), dtype=torch.float64, device=b.device)

    @property
    def observation_space(self):
        sp = super().observation_space
        return spaces.Box(0.0, 255.0, sp.shape, dtype=np.float64)

    def step(self, actions, **kw):
        import torch
        b = self.batched
        st = b._stream()
        for k in range(self.frame_skip):
            b.sim.render(self._window[k].data_ptr(), st)                    # obs = env.render_obs(); window.append(obs)
            _, rew, done, info = b.step(actions, render=False)              # env.update_physics(action)
        b.sim.render(self._window[3].data_ptr(), st)
        b.sim.blend4([w.data_ptr() for w in self._window], self.WEIGHTS, self._blurred.data_ptr(), self._blurred.numel(), st)
        return self._blurred, rew, done, info
