"""Seeded runs without the navigation task, recorded byte for byte: every step's frame (as a SHA-256 of the obs batch),
reward and done flags, the terminal frames, and the envs' streams and poses at the end.  tests/golden/nav_off_baseline.npz
holds these runs as the commit before DTS_FLAG_NAV made them; tests/test_gpu_nav.py holds every later tree to it, so
the flag changes nothing for a handle that does not set it.  Needs a GPU.

    python tests/nav_off_baseline.py <out.npz>      (records the tree it runs in)
"""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M64 = (1 << 64) - 1
# (tag, map(s), keywords, steps, host reset every `every` steps (0: auto-reset only))
RUNS = [
    ("auto", "small_loop", dict(domain_rand=True, device_reset=True, auto_reset=True, terminal_obs=True, max_steps=40,
                                dynamics_rand=True), 90, 0),
    ("dyn", "loop_dyn_duckiebots", dict(domain_rand=True, device_reset=True, auto_reset=True, max_steps=50), 70, 0),
    ("multi", ["small_loop", "udem1"], dict(domain_rand=False, device_reset=True, auto_reset=True, max_steps=30,
                                            randomize_maps_on_reset=True), 60, 0),
    ("host", "loop_obstacles", dict(domain_rand=True, device_reset=False, max_steps=1500), 30, 10),
]


def record():
    import torch
    sys.path.insert(0, ROOT)
    from gym_duckietown_b200.batched_env import BatchedDuckietownEnv
    out = {}
    for tag, maps_, kw, steps, every in RUNS:
        n = 48
        env = BatchedDuckietownEnv(n, maps_, camera_width=64, camera_height=48, seed=77, **kw)
        try:
            env.reset()
            acts = torch.from_numpy(np.random.default_rng(5).uniform(-1, 1, (steps, n, 2)).astype(np.float32)).cuda()
            acts[:, :, 0] = acts[:, :, 0].abs()
            sha, rew, done, term = [], [], [], []
            for t in range(steps):
                if every and t and t % every == 0:
                    env.reset()
                obs, r, d, _ = env.step(acts[t])
                torch.cuda.synchronize()
                sha.append(np.frombuffer(hashlib.sha256(obs.cpu().numpy().tobytes()).digest(), np.uint8))
                rew.append(r.cpu().numpy().copy())
                done.append(d.cpu().numpy().astype(np.uint8))
                if env.terminal_obs is not None:
                    term.append(np.frombuffer(hashlib.sha256(env.terminal_obs.cpu().numpy().tobytes()).digest(), np.uint8))
            st = {k: v.cpu().numpy() for k, v in env.state.items()}
            gens = env.sim.debug_streams() if env.device_reset else [g.bit_generator.state for g in env.sampler.rngs]
            out[f"{tag}_obs_sha"] = np.stack(sha)
            out[f"{tag}_reward"] = np.stack(rew)
            out[f"{tag}_done"] = np.stack(done)
            if term:
                out[f"{tag}_terminal_sha"] = np.stack(term)
            out[f"{tag}_streams"] = np.array([[g["state"]["state"] >> 64, g["state"]["state"] & M64, g["has_uint32"],
                                               g["uinteger"]] for g in gens], np.uint64)
            for k in ("pos_x", "pos_z", "angle", "step_count", "episode", "map_id", "done_code"):
                out[f"{tag}_{k}"] = st[k].copy()
        finally:
            env.close()
    return out


if __name__ == "__main__":
    np.savez_compressed(sys.argv[1], **record())
    print("recorded", sys.argv[1])
