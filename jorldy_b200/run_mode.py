"""Run modes with the reference's entry points (jorldy/run_mode.py:10,106,212,366).

single_train            the reference's own per-step loop (run_mode.py:68-91) over the numpy plugin API,
                        one env — kept so `--single` behaves exactly as before, only the arithmetic moved
                        to the GPU.
sync_distributed_train  the GPU-resident pipeline that replaces ray actors + the sync gather
                        (run_mode.py:163-198, manager/distributed_manager.py): `train.num_workers` becomes the
                        number of batched env instances stepped by one kernel; on-policy agents use
                        RolloutCollector (+ learn_rollout), REINFORCE EpisodeCollector (+ learn_episodes),
                        replay agents use ReplayCollector.  Under torchrun
                        every rank runs this loop on its own GPU with gradient all-reduce (core/parallel.py).
async_distributed_train same pipeline (there is no separate interact process to be asynchronous with:
                        collection and learning share the device; Ape-X per-actor epsilons are per env row).
evaluate                greedy episodes from a checkpoint (run_mode.py:366-402).
"""
import os
import time
import traceback

import numpy as np
import torch

from .core import Agent, Env
from .core.collect import EpisodeCollector, ReplayCollector, RolloutCollector
from .manager import ConfigManager, LogManager, MetricManager


def _agent_config(config, env, **extra):
    cfg = {"state_size": env.state_size, "action_size": env.action_size, "optim_config": config.optim,
           "run_step": config.train.run_step}
    cfg.update(extra)
    cfg.update(config.agent)
    return cfg


def _attach_legal(env, agent):
    """Board games: an agent that masks illegal moves (MuZero) reads the env's legal-move mask in place."""
    if hasattr(env, "legal") and hasattr(agent, "attach_legal"):
        agent.attach_legal(env.legal)


def _check_players(env, agent):
    """A two-player env (TicTacToe self-play) needs an agent whose targets alternate sides (MuZero two_player=True),
    and such an agent needs a two-player env: any other pairing would learn from values of the wrong sign."""
    env_2p, agent_2p = getattr(env, "two_player", False), getattr(agent, "two_player", False)
    if env_2p != agent_2p:
        raise ValueError(f"{type(env).__name__} is {'a two-player' if env_2p else 'a single-agent'} env but "
                         f"{type(agent).__name__} was built for {'two players' if agent_2p else 'a single agent'}: "
                         "two-player self-play takes MuZero with two_player=True")


def _report(step, metrics, logger, env, t0):
    stat = metrics.get_statistics()
    ep, sc = env.stats.tolist()
    if ep > 0:
        stat["score"] = round(sc / ep, 4)
        env.stats.zero_()
    stat["steps_per_sec"] = round(step / max(time.time() - t0, 1e-9), 1)
    print(f"{step} step | " + " | ".join(f"{k}: {v}" for k, v in stat.items()), flush=True)
    logger.write({k: v for k, v in stat.items() if isinstance(v, (int, float))}, step)


def single_train(config_path, unknown):
    config_manager = ConfigManager(config_path, unknown)
    config = config_manager.config
    env = Env(**config.env)
    agent = Agent(**_agent_config(config, env))
    assert agent.action_type == env.action_type
    if config.train.load_path:
        agent.load(config.train.load_path)
    _check_players(env, agent)
    _attach_legal(env, agent)
    logger = LogManager(config.env.name, config.train.id or config.agent.name, config.train.experiment)
    config_manager.dump(logger.path)
    metrics = MetricManager()
    t0 = time.time()
    try:
        state = env.reset()
        for step in range(1, config.train.run_step + 1):
            action_dict = agent.act(state, config.train.training)
            next_state, reward, done = env.step(action_dict["action"])
            transition = {"state": state, "next_state": next_state, "reward": reward, "done": done}
            transition.update(action_dict)
            transition = agent.interact_callback(transition)
            if transition:
                result = agent.process([transition], step)
                if result:
                    metrics.append(result)
            if done:
                metrics.append({"score": env.score})
            if step % config.train.print_period == 0 or step == config.train.run_step:
                stat = metrics.get_statistics()
                print(f"{step} step | " + " | ".join(f"{k}: {v}" for k, v in stat.items()), flush=True)
                logger.write(stat, step)
            if step % config.train.save_period == 0 or step == config.train.run_step:
                agent.save(logger.path)
            state = next_state if not done else env.reset()
    except Exception:
        traceback.print_exc()
    finally:
        env.close()


def sync_distributed_train(config_path, unknown):
    config_manager = ConfigManager(config_path, unknown)
    config = config_manager.config
    rank = int(os.environ.get("RANK", 0))
    world = int(os.environ.get("WORLD_SIZE", 1))
    local_rank = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local_rank)
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    num_envs = int(config.train.num_workers or 1)
    env = Env(**config.env, num_envs=num_envs, id=rank, seed=int(config.train.seed or 0))
    extra = {"num_workers": num_envs * world}
    cfg = _agent_config(config, env, **extra)
    if config.train.distributed_batch_size:
        cfg["batch_size"] = config.train.distributed_batch_size      # run_mode.py:121-122
    agent = Agent(**cfg)
    assert agent.action_type == env.action_type
    if config.train.load_path:
        agent.load(config.train.load_path)
    _check_players(env, agent)
    _attach_legal(env, agent)
    if world > 1:
        from .core import parallel
        parallel.attach(agent, world)
    logger = metrics = None
    if rank == 0:
        logger = LogManager(config.env.name, config.train.id or config.agent.name, config.train.experiment)
        config_manager.dump(logger.path)
        metrics = MetricManager()
    on_policy = hasattr(agent, "learn_rollout")
    episodic = hasattr(agent, "learn_episodes")        # REINFORCE: whole episodes from an episode ring
    update_period = int(config.train.update_period or getattr(agent, "n_step", 1))
    if episodic:
        collector = EpisodeCollector(env, agent, update_period)
    else:
        collector = RolloutCollector(env, agent) if on_policy else ReplayCollector(env, agent, update_period)
    step, t0 = 0, time.time()
    next_print = config.train.print_period
    next_save = config.train.save_period
    try:
        while step < config.train.run_step:
            if episodic:
                result = agent.learn_episodes(collector.collect())
                step += collector.T
                if result and agent.lr_decay:            # a round that completed no episode learns nothing
                    agent.learning_rate_decay(step)
            elif on_policy:
                result = agent.learn_rollout(collector.collect())
                step += agent.n_step
                if agent.lr_decay:
                    agent.learning_rate_decay(step)
            else:
                step, result = collector.run_round(step)
            if rank == 0:
                if result:
                    metrics.append(result)
                if step >= next_print or step >= config.train.run_step:
                    _report(step, metrics, logger, env, t0)
                    next_print += config.train.print_period
                if step >= next_save or step >= config.train.run_step:
                    agent.save(logger.path)
                    next_save += config.train.save_period
    except Exception:
        traceback.print_exc()
    finally:
        env.close()
        if world > 1:
            import torch.distributed as dist
            dist.destroy_process_group()


def async_distributed_train(config_path, unknown):
    return sync_distributed_train(config_path, unknown)


def evaluate(config_path, unknown):
    config_manager = ConfigManager(config_path, unknown)
    config = config_manager.config
    env = Env(**config.env, train_mode=False)
    agent = Agent(**_agent_config(config, env))
    assert config.train.load_path
    agent.load(config.train.load_path)
    _check_players(env, agent)
    _attach_legal(env, agent)
    episode = 0
    state = env.reset()
    try:
        for step in range(1, config.train.run_step + 1):
            action_dict = agent.act(state, training=False)
            next_state, reward, done = env.step(action_dict["action"])
            if done:
                episode += 1
                print(f"{episode} Epi | {step} step | score: {env.score}")
            state = next_state if not done else env.reset()
    except Exception:
        traceback.print_exc()
    finally:
        env.close()
