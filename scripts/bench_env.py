"""Throughput of the device RL environment step (VectorEnv.step over b2s_env_step) at 2^20 lanes, beside the same time step
composed from the older calls: b2s_step_fused, one b2s_observation / b2s_information_state per player and, for poker, a
Python chance loop (b2s_status -> draw from the legal mask in torch -> b2s_apply_actions) with a host sync per chance node.
The composed step does not reset finished lanes (the batch API had no per-lane reset), so it is a lower bound on that
path's cost.  Prints the card and its power limit, then one JSON line per workload with the median and spread of
`--repeats` timed windows.

  python scripts/bench_env.py [--lanes 1048576] [--steps 50] [--warmup 10] [--repeats 3]

Times: env_step_device_s and k_env_step_s are kernel times from torch.profiler (k_env_step + the per-player k_obs + the
counter kernel; k_env_step alone); wall_s_per_step_with_policy are CUDA-event times of whole steps including the same
lowest-legal-action policy on both paths.  The composed path is timed over 4-step windows from fresh episodes.
Algorithmic bytes per lane and step: state_bytes (the lane blob size of b2s_game_info, which is at least the stored lane)
read + written, 4 action bytes read, outputs 4 * mask_words + 4 * P + 3 written, and per player an observation of 4 * F
bytes written plus the state read again by its k_obs launch.  Achieved GB/s = those bytes / kernel time; the share of peak
is against the H100 SXM data-sheet 3.35 TB/s."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import open_spiel_b200 as b2  # noqa: E402
from open_spiel_b200._lib import EnvOut, check, lib  # noqa: E402

PEAK_BYTES = 3.35e12
WORKLOADS = [("connect_four", None), ("leduc_poker", "INFORMATION_STATE"), ("go(board_size=9)", None)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def lowest_legal(mask):
    return mask.to(torch.int32).argmax(1).to(torch.int32)


def time_windows(fn, steps, warmup, repeats, before=None):
    """Seconds per call of fn over `repeats` windows of `steps` calls (CUDA events), sorted."""
    for _ in range(warmup):
        fn()
    out = []
    for _ in range(repeats):
        if before:
            before()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(steps):
            fn()
        b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b) / 1e3 / steps)
    return sorted(out)


def kernel_times(fn, steps):
    """Device seconds per call of fn by kernel name (torch.profiler, CUDA activity), over `steps` calls."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        out[e.key] = out.get(e.key, 0.0) + t / 1e6 / steps
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lanes", type=int, default=1 << 20)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_env.py measures on a CUDA device"
    print("card:", card(), flush=True)
    n = args.lanes
    for gs, kind in WORKLOADS:
        env = b2.VectorEnv(gs, n, seed=1, observation_type=kind)
        info = env.batch.info
        P, W, F = info.num_players, info.mask_words, env._obs.shape[2]
        env.reset()
        acts = torch.zeros(n, dtype=torch.int32, device="cuda")

        def env_step():
            acts.copy_(lowest_legal(env.time_step.legal_actions_mask))
            env.step(acts, reset_if_done=True)

        t_env = time_windows(env_step, args.steps, args.warmup, args.repeats)
        dev = kernel_times(env_step, args.steps)
        t_env_dev = sum(v for k, v in dev.items() if "k_env_step" in k or "k_obs" in k or "k_env_tick" in k)
        t_kernel = sum(v for k, v in dev.items() if "k_env_step" in k)

        # the composed step from the older calls on a plain batch
        batch = b2.load_game(gs).new_batch(n)
        mask_w = torch.empty((n, W), dtype=torch.int32, device="cuda")
        term = torch.empty(n, dtype=torch.uint8, device="cuda")
        rets = torch.empty((n, P), dtype=torch.float32, device="cuda")
        obs = torch.empty((P, n, F), dtype=torch.float32, device="cuda")
        chance = info.max_chance_outcomes > 0
        gen = torch.Generator(device="cuda").manual_seed(0)
        bits = torch.arange(32, dtype=torch.int32, device="cuda")

        def resolve_chance():
            while True:
                cur, _, _ = batch.status()
                at_chance = cur == -1
                if not bool(at_chance.any()):                       # host sync per chance node
                    return
                m = ((batch.legal_actions_mask_words() .unsqueeze(-1) >> bits) & 1).reshape(n, -1).to(torch.int32)
                cnt = m.sum(1)
                k = (torch.rand(n, device="cuda", generator=gen) * cnt).to(torch.int32)
                a = (m.cumsum(1) <= k.unsqueeze(1)).sum(1).to(torch.int32)
                batch.apply_actions(torch.where(at_chance, a, torch.full_like(a, -1)).contiguous())

        def restart():              # every window starts from fresh episodes: the composed path cannot reset single lanes
            batch.reset()
            if chance:
                resolve_chance()
            batch.step(torch.full((n,), -1, dtype=torch.int32, device="cuda"), mask_w, term, rets)

        def composed_step():
            dense = ((mask_w.unsqueeze(-1) >> bits) & 1).reshape(n, -1)[:, :info.num_distinct_actions]
            a = lowest_legal(dense)
            a = torch.where(term.bool(), torch.full_like(a, -1), a).contiguous()
            batch.step(a, mask_w, term, rets)
            if chance:
                resolve_chance()
                batch.legal_actions_mask_words(out=mask_w)
            for p in range(P):
                if kind == "INFORMATION_STATE":
                    batch.information_state_tensor(p, out=obs[p])
                else:
                    batch.observation_tensor(p, out=obs[p])

        t_comp = time_windows(composed_step, 4, 0, args.repeats, before=restart)
        sb = info.state_bytes
        bytes_step = n * (2 * sb + 4 + 4 * W + 4 * P + 3 + P * (sb + 4 * F))
        bytes_kernel = n * (2 * sb + 4 + 4 * W + 4 * P + 3)
        med = lambda t: t[len(t) // 2]  # noqa: E731
        spread = lambda t: {"median": med(t), "min": t[0], "max": t[-1]}  # noqa: E731
        print(json.dumps({
            "game": gs, "observation": kind or "default", "lanes": n, "players": P, "tensor_floats": F, "state_bytes": sb,
            "env_step_device_s": t_env_dev, "env_steps_per_s": n / t_env_dev,
            "bytes_per_step": bytes_step, "step_GBps": bytes_step / t_env_dev / 1e9, "step_peak_share": bytes_step / t_env_dev / PEAK_BYTES,
            "k_env_step_s": t_kernel, "k_env_step_bytes": bytes_kernel, "k_env_step_GBps": bytes_kernel / t_kernel / 1e9,
            "k_env_step_peak_share": bytes_kernel / t_kernel / PEAK_BYTES,
            "wall_s_per_step_with_policy": {"env_step": spread(t_env), "composed": spread(t_comp)},
            "wall_speedup_vs_composed": med(t_comp) / med(t_env),
        }), flush=True)
        del env, batch, obs
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
