"""What saving and loading the envs' state costs (BatchedDuckietownEnv.save_state / load_state).

For each map (c2: small_loop; loop_dyn_duckiebots, whose records also carry its obstacles), at 4096 envs x 160x120:
the record size, and the time of one dts_save_state and one dts_load_state (all envs) from CUDA events around
`repeats` back-to-back calls after `warmup` calls: issued one by one from Python ("eager", which the host's call rate
may bound), and replayed from a CUDA graph of the same calls ("device").  Bytes moved per call count the state read
and the records written (or the reverse): 2 x num_envs x record_bytes.  Prints one JSON line, with the card's name and
power limit read in the same run.

    python tools/state_probe.py [--envs 4096] [--repeats 200] [--warmup 20] [--out FILE.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gym_duckietown_b200.batched_env import BatchedDuckietownEnv  # noqa: E402

MAPS = {"c2": "small_loop", "dyn": "loop_dyn_duckiebots"}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def timed_ms(fn, repeats, warmup):
    """(eager, graph) milliseconds per call of `fn`, which launches on the current stream."""
    for _ in range(warmup):
        fn()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(repeats):
        fn()
    end.record()
    end.synchronize()
    eager = start.elapsed_time(end) / repeats
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(repeats):
            fn()
    graph.replay()
    torch.cuda.synchronize()
    start.record()
    graph.replay()
    end.record()
    end.synchronize()
    return eager, start.elapsed_time(end) / repeats


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--repeats", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    res = {"card": card(), "envs": a.envs, "repeats": a.repeats, "camera": "160x120", "configs": {}}
    for cfg, name in MAPS.items():
        env = BatchedDuckietownEnv(a.envs, name, camera_width=160, camera_height=120, domain_rand=False, seed=1,
                                   device_reset=True, auto_reset=True)
        env.reset()
        g = torch.Generator(device="cuda").manual_seed(0)
        for _ in range(10):
            env.step(torch.rand((a.envs, 2), device="cuda", generator=g) * 2 - 1)
        rec = env.save_state()
        fp = rec.fingerprint
        save = timed_ms(lambda: env.save_state(out=rec), a.repeats, a.warmup)
        load = timed_ms(lambda: env.load_state(rec, fingerprint=fp), a.repeats, a.warmup)
        env.check()
        moved = 2 * a.envs * rec.shape[1]
        out = {"map": name, "record_bytes": int(rec.shape[1]), "bytes_per_call": moved}
        for what, (eager, dev) in (("save", save), ("load", load)):
            out[f"{what}_us_eager"], out[f"{what}_us_device"] = eager * 1e3, dev * 1e3
            out[f"{what}_gbs_device"] = moved / (dev * 1e-3) / 1e9
        res["configs"][cfg] = out
        print(f"{cfg}: {res['configs'][cfg]}", file=sys.stderr, flush=True)
        env.close()
        del env
        torch.cuda.empty_cache()
    res["card_after"] = card()
    line = json.dumps(res)
    print(line, flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
