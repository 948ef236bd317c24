"""Eager against device rollout storage (soundspaces_b200/rollout.py), alternated in one run, at the trainers' shapes:
num_steps 150; N = 5, 10 and 16; AV-Nav (spectrogram, depth, hidden 512), AV-WaN (the same plus gm, am and action_map)
and SAVi with its external memory at the SCENE_MEMORY_TRANSFORMER sizes (memory_size 150 + num_steps slots, capacity
150, 256 wide; 2 minibatches where N is even, else 1).  The inputs are what the stock trainers pass: AV-Nav and AV-WaN
call ``batch_obs(observations)`` without a device, so every sensor but this project's device-rendered spectrogram
arrives on the CPU, and they build rewards and masks on the CPU; SAVi's trainer passes a device batch, rewards and
masks.  The eager side is tests/rollout_models.py's stand-ins of the reference classes.

Per config it reports the time per insert (150 inserts, host clock to a device synchronise, divided by 150), the time
of compute_returns + get_advantages + one full generator pass + after_update, and the storage-only env-steps/s of a
150-step rollout (N * 150 over the inserts' time).  Then a 150-step AV-Nav-style rollout loop on the trace-replay env
(replay.py, 16 envs, 8x8 scene, 16 kHz): policy act, env step, ``batch_obs`` into the spectrogram slot, rewards and
masks built on the CPU, ``insert``, then the update above; env-steps/s of the whole loop with each storage.  Median of
--reps alternated repetitions.  Prints the card's name and power limit and one JSON line per measurement.

    python scratch/rollout_storage_bench.py [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import rollout_models as rm  # noqa: E402
from soundspaces_b200 import rollout as ro  # noqa: E402

S = 150
DEV = torch.device("cuda", 0)
CONFIGS = {
    "av_nav": dict(kind="common", sensors={"spectrogram": (65, 26, 2), "depth": (128, 128, 1)}, mb=1, host=True),
    "av_wan": dict(kind="common", sensors={"spectrogram": (65, 26, 2), "depth": (128, 128, 1), "gm": (200, 200, 2),
                                           "am": (20, 20, 1), "action_map": (9, 9, 1)}, mb=1, host=True),
    "savi": dict(kind="savi", sensors={"spectrogram": (65, 26, 2), "depth": (128, 128, 1), "category": (21,)},
                 em=(150 + S, 150, 256), mb=2, host=False),
}
EAGER = dict(common=rm.CommonRolloutStorage, savi=rm.SaviRolloutStorage)
PATCHED = {k: ro.patch_rollout_storage(type("Patched" + v.__name__, (v,), {})) for k, v in EAGER.items()}
PATCHED_PPO = ro.patch_ppo(type("PatchedPPO", (rm.PPO,), {}))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def inputs(cfg, N):
    script = dict(kind=cfg["kind"], N=N, S=S, sensors=cfg["sensors"], layers=1, hidden=512, em=cfg.get("em"),
                  done_p=0.02, seed=0)
    g = np.random.default_rng(0)
    steps = []
    for _ in range(S):
        args = rm.to_device(rm.step_inputs(script, g), DEV, cfg["host"])
        if cfg["host"]:                                  # this project's batch_obs renders the spectrogram on the device
            args[0]["spectrogram"] = args[0]["spectrogram"].to(DEV)
        steps.append(args)
    return script, steps


def rollout(st, steps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for args in steps:
        st.insert(*args)
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def update(st, ppo, N, mb):
    nv = torch.zeros((N, 1), device=DEV)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    st.compute_returns(nv, True, 0.99, 0.95)
    adv = ppo.get_advantages(st)
    for batch in st.recurrent_generator(adv, mb):
        pass
    st.after_update()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def replay_loop(reps, N=16):
    """env-steps/s of a 150-step AV-Nav-style rollout plus its update on the trace-replay env, per storage."""
    from soundspaces_b200.replay import AudioPolicy, ReplayScene, ReplaySim, ReplayVectorEnv
    from soundspaces_b200.sensors import batch_obs
    from soundspaces_b200.simulator import AudioRenderService
    from synth import make_rir, make_source
    sr, taps = 16000, 16000
    svc = AudioRenderService(sr, device=DEV, max_taps=taps, n_terms=1)
    scene = ReplayScene("apartment_replay", side=8)
    rng = np.random.default_rng(11)
    base = np.stack([make_rir(500 + i, taps) for i in range(8)])
    mix = rng.standard_normal((4, scene.n_nodes, 8)).astype(np.float32) / 3.0
    scene.register_rirs(svc, source=0, rirs=np.einsum("anb,ble->anle", mix, base).astype(np.float32))
    clip = make_source(21, sr)
    sims = [ReplaySim(svc, scene, "telephone.wav", clip, source_node=0, start_node=int(rng.integers(scene.n_nodes)),
                      start_rotation=int(rng.integers(4)) * 90) for _ in range(N)]
    envs = ReplayVectorEnv(sims)
    spec = svc.renderer.spec_shape
    policy = AudioPolicy(spec).to(DEV)
    script = dict(kind="common", N=N, S=S, sensors={"spectrogram": spec}, layers=1, hidden=512)
    stores = {"eager": rm.make_storage(script, EAGER, DEV), "device": rm.make_storage(script, PATCHED, DEV)}
    ppo = {"eager": rm.PPO(), "device": PATCHED_PPO()}
    trace = rng.choice([1, 1, 1, 2, 3], size=(S, N))
    hidden = torch.zeros((1, N, 512), device=DEV)

    def one(st, k):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        batch_obs(envs.observe(), device=DEV, out={"spectrogram": st.observations["spectrogram"][0]})
        for step in range(S):
            with torch.no_grad():
                value, actions, log_probs = policy.act(st.observations["spectrogram"][step], fused=True)
            acts = trace[step].tolist()
            observations = envs.step(acts)
            batch = batch_obs(observations, device=DEV,
                              out={"spectrogram": st.observations["spectrogram"][st.step + 1]})
            batch = {key: batch[key] for key in st.observations}
            rewards = torch.tensor([[0.1 * a] for a in acts], dtype=torch.float)       # built on the CPU
            masks = torch.tensor([[1.0] for _ in acts], dtype=torch.float)
            st.insert(batch, hidden, actions.view(N, 1), log_probs.view(N, 1), value.view(N, 1), rewards, masks)
        update(st, ppo[k], N, 1)
        return time.perf_counter() - t0

    t = {k: [] for k in stores}
    for rep in range(reps + 1):
        for k, st in stores.items():
            w = one(st, k)
            if rep:
                t[k].append(w)
    med = lambda xs: sorted(xs)[len(xs) // 2]  # noqa: E731
    res = {"config": "trace_replay_av_nav_loop", "N": N, "num_steps": S, "reps": reps}
    for k in stores:
        res[f"{k}_rollout_ms"] = round(med(t[k]) * 1e3, 1)
        res[f"{k}_env_steps_per_s"] = round(N * S / med(t[k]))
    res["speedup"] = round(res["eager_rollout_ms"] / res["device_rollout_ms"], 3)
    print(json.dumps(res), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--envs", default="5,10,16")
    args = ap.parse_args()
    print("card:", card(), flush=True)
    ppo = {"eager": rm.PPO(), "device": PATCHED_PPO()}
    for name, cfg in CONFIGS.items():
        for N in map(int, args.envs.split(",")):
            script, steps = inputs(cfg, N)
            stores = {"eager": rm.make_storage(script, EAGER, DEV), "device": rm.make_storage(script, PATCHED, DEV)}
            t = {k: {"insert": [], "update": []} for k in stores}
            for rep in range(args.reps + 1):                       # rep 0 warms up
                for k, st in stores.items():
                    ti = rollout(st, steps)
                    tu = update(st, ppo[k], N, cfg["mb"] if N % cfg["mb"] == 0 else 1)
                    if rep:
                        t[k]["insert"].append(ti / S)
                        t[k]["update"].append(tu)
            med = lambda xs: sorted(xs)[len(xs) // 2]  # noqa: E731
            res = {"config": name, "N": N, "num_steps": S, "reps": args.reps}
            for k in stores:
                res[f"{k}_insert_us"] = round(med(t[k]["insert"]) * 1e6, 1)
                res[f"{k}_update_ms"] = round(med(t[k]["update"]) * 1e3, 3)
                res[f"{k}_env_steps_per_s"] = round(N / med(t[k]["insert"]))
            res["insert_speedup"] = round(res["eager_insert_us"] / res["device_insert_us"], 2)
            res["update_speedup"] = round(res["eager_update_ms"] / res["device_update_ms"], 2)
            print(json.dumps(res), flush=True)
            del stores
            torch.cuda.empty_cache()
    replay_loop(args.reps)


if __name__ == "__main__":
    main()
