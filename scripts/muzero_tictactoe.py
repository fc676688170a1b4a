"""Does MuZero learn TicTacToe?  Trains --config (default `config.muzero.tictactoe`: 8 envs, S = 50, against the
uniform-random opponent; `config.muzero.tictactoe_selfplay` trains by two-player self-play) from a fixed seed for
--steps batched env steps (the step count of `main --sync`: one act over all 8 envs each; a self-play step is one ply,
a random-opponent step a move and the reply) under the batched collector.  Before and after training it reports:
  - untrained / trained: the win / draw / loss / forfeit rates of --games greedy games against the random opponent;
  - untrained_perfect / trained_perfect: the same against the perfect opponent (opponent="perfect"), split by whether
    the agent moved first;
  - untrained_optimal_move_rate / trained_optimal_move_rate: the share of the 4 520 non-terminal positions where the
    greedy masked search (one act over all of them, from the side to move) picks a move that keeps the position's
    negamax value (core/env/tictactoe.py solve()).
Also reports the median act, collection-round and learn times from device events after the first --warmup calls of
each, and the card's name and power limit, read in the same run.  Prints one JSON line.

    python scripts/muzero_tictactoe.py [--config config.muzero.tictactoe] [--steps 60000] [--games 10000] [--seed 0]
                                       [--warmup 50]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def _rates(o, f):
    return {"win": float(np.mean(o == 1)), "draw": float(np.mean(o == 0)), "loss": float(np.mean((o == -1) & ~f)),
            "forfeit": float(np.mean(f))}


def play(agent, games, seed, opponent="random"):
    """`games` greedy games at once, one board each, without auto-reset: the first done of each board is its outcome.
    Against the perfect opponent the rates are split by whether the agent moved first."""
    from jorldy_b200.core import Env
    env = Env("tictactoe", num_envs=games, seed=seed, id=7, auto_reset=False, opponent=opponent)
    env.reset_device()
    first = (env.obs[:, 9:].sum(1) == 0).cpu().numpy()        # the opponent did not open
    agent.attach_legal(env.legal)
    live = torch.ones(games, dtype=torch.bool, device="cuda")
    forfeit = torch.zeros(games, dtype=torch.bool, device="cuda")
    outcome = torch.zeros(games, device="cuda")
    for _ in range(env.max_steps):
        a, _ = agent.act_device(env.obs, training=False)
        forfeit |= live & (env.legal.gather(1, a.view(-1, 1)).view(-1) == 0)
        env.step_device(a)
        outcome = torch.where(live & (env.done > 0), env.reward, outcome)
        live &= env.done == 0
    assert not bool(live.any())
    f, o = forfeit.cpu().numpy(), outcome.cpu().numpy()
    if opponent == "random":
        return _rates(o, f)
    return {"moved_first": dict(_rates(o[first], f[first]), games=int(first.sum())),
            "moved_second": dict(_rates(o[~first], f[~first]), games=int((~first).sum()))}


def optimal_move_rate(agent):
    """One greedy act over the 4 520 non-terminal positions (obs and legal moves from the side to move); the share of
    them where the action reaches the position's negamax value."""
    from jorldy_b200.core.env.tictactoe import position, solve
    best = solve()[1]
    pos = [(m, o) for m in range(512) for o in range(512) if not m & o and best[position(m, o)]]
    bits = np.array([[(m >> c) & 1 for c in range(9)] + [(o >> c) & 1 for c in range(9)] for m, o in pos],
                    dtype=np.float32)
    obs = torch.as_tensor(bits, device="cuda")
    legal = (1 - obs[:, :9] - obs[:, 9:]).to(torch.uint8).contiguous()
    agent.attach_legal(legal)
    a, _ = agent.act_device(obs, training=False)
    a = a.cpu().numpy()
    masks = np.array([best[position(m, o)] for m, o in pos])
    return {"positions": len(pos), "rate": float(np.mean((masks >> a) & 1))}


def evaluate(agent, games, seed):
    return {"random": play(agent, games, seed), "perfect": play(agent, games, seed + 1, "perfect"),
            "optimal_move_rate": optimal_move_rate(agent)}


class Timed:
    """Wraps a bound method: a device event pair around every call."""

    def __init__(self, fn):
        self.fn, self.events = fn, []

    def __call__(self, *a, **kw):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = self.fn(*a, **kw)
        e1.record()
        self.events.append((e0, e1))
        return out

    def median_ms(self, warmup):
        t = [a.elapsed_time(b) for a, b in self.events[warmup:]]
        return float(np.median(t)) if t else None, len(t)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="config.muzero.tictactoe")
    ap.add_argument("--steps", type=int, default=60000)
    ap.add_argument("--games", type=int, default=10000)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--warmup", type=int, default=50)
    args = ap.parse_args()
    from jorldy_b200 import config as cfg
    from jorldy_b200.core import Agent, Env
    from jorldy_b200.core.collect import ReplayCollector
    c = cfg.load(args.config)
    env = Env(**c.env, num_envs=c.train["num_workers"], seed=args.seed)
    agent = Agent(**c.agent, state_size=env.state_size, action_size=env.action_size, optim_config=c.optim,
                  run_step=args.steps, num_workers=env.num_envs, device="cuda", seed=args.seed)
    before = evaluate(agent, args.games, seed=1000 + args.seed)
    agent.attach_legal(env.legal)
    col = ReplayCollector(env, agent, c.train["update_period"])
    agent.act_device, agent.learn = Timed(agent.act_device), Timed(agent.learn)
    rounds = Timed(col.run_round)
    step, t0, learns = 0, time.time(), 0
    while step < args.steps:
        step, res = rounds(step)
        learns += bool(res)
        if res and agent.lr_decay:
            agent.learning_rate_decay(step)
    torch.cuda.synchronize()
    wall = time.time() - t0
    act_ms, n_act = agent.act_device.median_ms(args.warmup)
    round_ms, n_round = rounds.median_ms(args.warmup)
    learn_ms, n_learn = agent.learn.median_ms(args.warmup)
    ep, sc = env.stats.tolist()
    agent.act_device, agent.learn = agent.act_device.fn, agent.learn.fn
    after = evaluate(agent, args.games, seed=2000 + args.seed)
    print(json.dumps({"card": card(), "config": args.config, "seed": args.seed, "steps": step,
                      "env_steps": step * env.num_envs, "envs": env.num_envs, "num_simulation": agent.S, "learns": learns, "train_wall_s": round(wall, 1),
                      "train_episodes": ep, "train_mean_score": sc / ep if ep else None, "games": args.games,
                      "untrained": before["random"], "trained": after["random"],
                      "untrained_perfect": before["perfect"], "trained_perfect": after["perfect"],
                      "untrained_optimal_move_rate": before["optimal_move_rate"],
                      "trained_optimal_move_rate": after["optimal_move_rate"],
                      "median_ms": {"act": act_ms, "round": round_ms, "learn": learn_ms},
                      "timed_calls": {"act": n_act, "round": n_round, "learn": n_learn}}))


if __name__ == "__main__":
    main()
