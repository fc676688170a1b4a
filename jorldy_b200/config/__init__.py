"""Built-in hot-path configs, generated from tables instead of one file per (agent, env) pair.

`load("config.<agent>.<env>")` returns a module-like namespace with the four dicts the reference's
config modules define (jorldy/config/<agent>/<env>.py: env / agent / optim / train).  Values follow the
reference's shipped configs for the agents on the north-star path (dqn, double, dueling, multistep,
per, noisy, c51, rainbow, qrdqn, iqn, m_dqn, m_iqn, rainbow_iqn, ape_x, r2d2, ppo, and ddpg / td3 / sac of SURVEY 8f-4) on cartpole / mountaincar /
pendulum / atari(synthetic) / mujoco(synthetic dims), plus the discrete-action SAC's `config.sac_discrete.{cartpole,atari}` (agent name "sac"),
which follow the SAC-Discrete paper, and `config.vmpo.{cartpole,mountaincar,pendulum,mujoco,atari}`, PPO's rows with the V-MPO
paper's multiplier settings, `config.icm_ppo.{cartpole,mountaincar,pendulum,mujoco,atari}`, PPO's rows with the ICM keys,
`config.rnd_ppo.{cartpole,mountaincar,pendulum,mujoco,atari}`, PPO's rows with the RND keys,
`config.mpo.{cartpole,mountaincar,pendulum,mujoco}`, this project's MPO settings on SAC's replay rows, and
`config.reinforce.{cartpole,mountaincar,pendulum,mujoco}`, PPO's rows with the REINFORCE keys, and
`config.muzero.{cartpole,mountaincar,atari,tictactoe,tictactoe_selfplay}`, this project's MuZero settings; an existing JORLDY config directory on sys.path takes precedence
(manager/config_manager.py).
"""
from types import SimpleNamespace

_TRAIN_SMALL = dict(training=True, load_path=None, run_step=100000, print_period=1000, save_period=10000)
_TRAIN_ATARI = dict(training=True, load_path=None, run_step=30000000, print_period=10000, save_period=100000,
                    eval_iteration=5, eval_time_limit=None, record=True, record_period=300000)
_EPS = dict(epsilon_init=1.0, epsilon_min=0.01, explore_ratio=0.2)
_REPLAY = dict(gamma=0.99, buffer_size=50000, batch_size=32, start_train_step=2000, target_update_period=500, lr_decay=True)
_REPLAY_ATARI = dict(gamma=0.99, buffer_size=1000000, batch_size=32, start_train_step=100000,
                     target_update_period=10000, lr_decay=True, head="cnn")
_ATARI_ENV = dict(render=False, gray_img=True, img_width=84, img_height=84, stack_frame=4, no_op=True, skip_frame=4,
                  reward_clip=True, episodic_life=True)

# agent name -> (network, extra agent keys, eval_iteration, update_period on cartpole)
_VALUE_AGENTS = {
    "dqn": ("discrete_q_network", dict(_EPS), 10, 32),
    "double": ("discrete_q_network", dict(_EPS), 5, 32),
    "dueling": ("dueling", dict(_EPS), 5, 32),
    "multistep": ("discrete_q_network", dict(_EPS, n_step=4), 5, 8),
    "per": ("discrete_q_network", dict(_EPS, alpha=0.6, beta=0.4, learn_period=2, uniform_sample_prob=1e-3), 5, 2),
    "noisy": ("noisy", dict(noise_type="factorized"), 5, 32),
    "c51": ("discrete_q_network", dict(_EPS, v_min=-1, v_max=10, num_support=51), 5, 32),
    "rainbow": ("rainbow", dict(n_step=3, alpha=0.5, beta=0.4, learn_period=2, uniform_sample_prob=1e-3,
                                noise_type="factorized", v_min=-1, v_max=10, num_support=51), 10, 8),
    # quantile agents (arXiv:1710.10044, arXiv:1806.06923): DQN's keys plus the papers' quantile counts
    "qrdqn": ("discrete_q_network", dict(_EPS, num_support=200), 10, 32),
    "iqn": ("iqn", dict(_EPS, num_sample=64, embedding_dim=64, sample_min=0.0, sample_max=1.0), 10, 32),
    # Munchausen agents (arXiv:2007.14430): DQN's / IQN's rows plus the paper's alpha, tau and l_0
    "m_dqn": ("discrete_q_network", dict(_EPS, alpha=0.9, tau=0.03, l_0=-1), 10, 32),
    "m_iqn": ("iqn", dict(_EPS, num_sample=64, embedding_dim=64, sample_min=0.0, sample_max=1.0, alpha=0.9, tau=0.03, l_0=-1),
              10, 32),
    # Rainbow-IQN (arXiv:1908.04683): Rainbow's row without the support, plus IQN's fraction counts; not compared with the
    # reference's config/rainbow_iqn/*.py, which takes precedence when a JORLDY config directory is on sys.path
    "rainbow_iqn": ("rainbow_iqn", dict(n_step=3, alpha=0.5, beta=0.4, learn_period=2, uniform_sample_prob=1e-3,
                                        noise_type="factorized", num_sample=64, embedding_dim=64, sample_min=0.0,
                                        sample_max=1.0), 10, 8),
}
_RAINBOW_ATARI = ("rainbow", "rainbow_iqn")      # learn_period 4, lr 2.5e-4 / 4 and 30 M steps on Atari


def _value_config(agent, env):
    net, extra, eval_it, upd = _VALUE_AGENTS[agent]
    if env == "atari":
        a = dict(name=agent, network=net, **_REPLAY_ATARI)
        a.update(extra)
        if "epsilon_min" in a:
            a.update(epsilon_min=0.1, explore_ratio=0.1)
        if agent in _RAINBOW_ATARI:
            a.update(learn_period=4)
        lr = 2.5e-4 / 4 if agent in _RAINBOW_ATARI else 1e-4
        return dict(env=dict(_ATARI_ENV), agent=a, optim=dict(name="adam", lr=lr),
                    train=dict(_TRAIN_ATARI, run_step=30000000 if agent in _RAINBOW_ATARI else 10000000,
                               update_period=32, num_workers=16))
    a = dict(name=agent, network=net, **_REPLAY)
    a.update(extra)
    env_d = dict(name="cartpole", action_type="discrete", render=False) if env == "cartpole" else dict(name="mountain_car", render=False)
    return dict(env=env_d, agent=a, optim=dict(name="adam", lr=1e-4),
                train=dict(_TRAIN_SMALL, eval_iteration=eval_it, update_period=upd, num_workers=8))


def _ape_x_config(env):
    a = dict(name="ape_x", network="dueling", gamma=0.99, clip_grad_norm=40.0, lr_decay=True, n_step=3, alpha=0.6,
             beta=0.4, uniform_sample_prob=1e-3, batch_size=32)
    opt = dict(name="rmsprop", eps=1.5e-7, centered=True)
    if env == "atari":
        a.update(head="cnn", buffer_size=2000000, start_train_step=50000, target_update_period=2500)
        return dict(env=dict(_ATARI_ENV), agent=a, optim=dict(opt, lr=2.5e-4 / 4),
                    train=dict(_TRAIN_ATARI, distributed_batch_size=512, update_period=100, num_workers=128))
    a.update(buffer_size=50000, start_train_step=2000, target_update_period=1000)
    env_d = dict(name="cartpole", action_type="discrete", render=False) if env == "cartpole" else dict(name="mountain_car", render=False)
    return dict(env=env_d, agent=a, optim=dict(opt, lr=1e-4),
                train=dict(_TRAIN_SMALL, eval_iteration=10, distributed_batch_size=512, update_period=16, num_workers=32))


def _r2d2_config(env):
    """R2D2 (Kapturowski et al., ICLR 2019).  atari: the paper's Table 2 (gamma 0.997, n 5, sequences of 80 with a burn-in
    of 40 stored every 40 steps, batch 64, Adam lr 1e-4 eps 1e-3, target period 2500, alpha 0.9, beta 0.6, eta 0.9, LSTM
    512, gradient clip 40), a replay of 100 000 sequences (4 M observations at stride 40) and Ape-X's actor epsilons.
    cartpole / mountaincar: Ape-X's row with seq_len 16, n_burn_in 8, n_step 4, eta 0.9, a choice of this project.  Not
    compared with the reference's config/r2d2/*.py, which takes precedence when a JORLDY config directory is on
    sys.path."""
    keys = dict(name="r2d2", network="r2d2", eta=0.9, zero_padding=True)
    if env == "atari":
        a = dict(keys, head="cnn", gamma=0.997, n_step=5, seq_len=80, n_burn_in=40, batch_size=64, buffer_size=100000,
                 start_train_step=50000, target_update_period=2500, alpha=0.9, beta=0.6, uniform_sample_prob=1e-3,
                 hidden_size=512, clip_grad_norm=40.0, lr_decay=True)
        return dict(env=dict(_ATARI_ENV), agent=a, optim=dict(name="adam", lr=1e-4, eps=1e-3),
                    train=dict(_TRAIN_ATARI, update_period=100, num_workers=128))
    d = _ape_x_config(env)
    d["agent"].update(keys, seq_len=16, n_burn_in=8, n_step=4)
    return d


def _ppo_config(env):
    a = dict(name="ppo", gamma=0.99, _lambda=0.95, epsilon_clip=0.1, vf_coef=1.0, ent_coef=0.01, clip_grad_norm=1.0,
             lr_decay=True)
    if env == "mujoco":
        a.update(network="continuous_policy_value", batch_size=512, n_step=2048, n_epoch=10)
        return dict(env=dict(render=False), agent=a, optim=dict(name="adam", lr=3e-4),
                    train=dict(training=True, load_path=None, run_step=1000000, print_period=10000, save_period=100000,
                               eval_iteration=10, record=True, record_period=500000, distributed_batch_size=2048,
                               update_period=2048, num_workers=32))
    a.update(batch_size=32, n_step=128, n_epoch=3, use_standardization=True)
    if env == "atari":
        # the PPO paper's Atari settings (as the cartpole config above uses); not compared key for key with the
        # reference's config/ppo/atari.py, which takes precedence when a JORLDY config directory is on sys.path
        a.update(network="discrete_policy_value", head="cnn")
        return dict(env=dict(_ATARI_ENV), agent=a, optim=dict(name="adam", lr=2.5e-4),
                    train=dict(_TRAIN_ATARI, run_step=30000000, eval_iteration=5, distributed_batch_size=256,
                               update_period=128, num_workers=8))
    if env == "pendulum":
        a.update(network="continuous_policy_value")
        env_d = dict(name="pendulum", render=False)
    elif env == "mountaincar":
        a.update(network="discrete_policy_value")
        env_d = dict(name="mountain_car", render=False)
    else:
        a.update(network="discrete_policy_value")
        env_d = dict(name="cartpole", action_type="discrete", render=False)
    return dict(env=env_d, agent=a, optim=dict(name="adam", lr=2.5e-4),
                train=dict(_TRAIN_SMALL, eval_iteration=10, distributed_batch_size=256, update_period=128, num_workers=8))


# V-MPO (Song et al., ICLR 2020, arXiv:1909.12238), keys added to _ppo_config's row for the same env.  The values come
# from the paper's hyper-parameter tables (Appendix): initial eta 1.0 in every table; discrete actions (DMLab / Atari
# tables): initial alpha 5.0, eps_eta 0.01, eps_alpha in [0.005, 0.01] -> 0.01; continuous control table: initial
# alpha_mu = alpha_sigma = 1.0, eps_eta 0.01, eps_alpha_mu in [0.005, 0.01] -> 0.005, eps_alpha_sigma in [5e-6, 5e-5]
# -> 5e-5.  The minima are 1e-8 (the multipliers stay positive).  alpha_sigma / eps_alpha_sigma are unused by discrete
# actions and kept at the continuous row's values.
_VMPO_KEYS = dict(min_eta=1e-8, min_alpha_mu=1e-8, min_alpha_sigma=1e-8, eta=1.0, alpha_sigma=1.0, eps_eta=0.01,
                  eps_alpha_sigma=5e-5)
_VMPO_ENVS = ("cartpole", "mountaincar", "pendulum", "mujoco", "atari")


def _vmpo_config(env):
    """V-MPO: PPO's config for the env (rollout, epochs, minibatch, GAE, clip_grad_norm, optimiser, train) plus the
    multiplier keys above.  Not compared with the reference's config/vmpo/*.py, which takes precedence when a JORLDY
    config directory is on sys.path."""
    d = _ppo_config(env)
    a = d["agent"]
    for k in ("epsilon_clip", "vf_coef", "ent_coef"):      # PPO's loss coefficients: no V-MPO counterpart
        a.pop(k)
    a.update(_VMPO_KEYS, name="vmpo")
    if a["network"].startswith("continuous"):
        a.update(alpha_mu=1.0, eps_alpha_mu=0.005)
    else:
        a.update(alpha_mu=5.0, eps_alpha_mu=0.01)
    return d


# ICM-PPO (Pathak et al., ICML 2017): keys added to _ppo_config's row for the same env, at the reference agent's
# constructor defaults.  Atari: the CNN ICM, without observation normalisation (not implemented for frames).
_ICM_PPO_KEYS = dict(icm_network="icm_mlp", beta=0.2, lamb=1.0, eta=0.01, extrinsic_coeff=1.0, intrinsic_coeff=1.0,
                     obs_normalize=True, ri_normalize=True, batch_norm=True)
_ICM_PPO_ENVS = ("cartpole", "mountaincar", "pendulum", "mujoco", "atari")


def _icm_ppo_config(env):
    """ICM-PPO: PPO's config for the env plus the ICM keys above."""
    d = _ppo_config(env)
    d["agent"].update(_ICM_PPO_KEYS, name="icm_ppo")
    if env == "atari":
        d["agent"].update(icm_network="icm_cnn", obs_normalize=False)
    return d


# RND-PPO (Burda et al., arXiv:1810.12894): keys added to _ppo_config's row for the same env, with the paper's advantage
# weights (extrinsic 2, intrinsic 1).  Atari: the CNN RND, without observation normalisation (not implemented for frames).
_RND_PPO_KEYS = dict(rnd_network="rnd_mlp", gamma_i=0.99, extrinsic_coeff=2.0, intrinsic_coeff=1.0, obs_normalize=True,
                     ri_normalize=True, batch_norm=True, non_episodic=True)
_RND_PPO_ENVS = ("cartpole", "mountaincar", "pendulum", "mujoco", "atari")


def _rnd_ppo_config(env):
    """RND-PPO: PPO's config for the env plus the RND keys above."""
    d = _ppo_config(env)
    d["agent"].update(_RND_PPO_KEYS, name="rnd_ppo")
    if env == "atari":
        d["agent"].update(rnd_network="rnd_cnn", obs_normalize=False)
    return d


# REINFORCE: PPO's env, optimiser and train rows for the same env without distributed_batch_size (REINFORCE has no
# minibatch), and PPO's network with the value head dropped.  These are this project's choices; a JORLDY config
# directory on sys.path takes precedence.
_REINFORCE_ENVS = ("cartpole", "mountaincar", "pendulum", "mujoco")


def _reinforce_config(env):
    d = _ppo_config(env)
    d["train"].pop("distributed_batch_size", None)
    d["agent"] = dict(name="reinforce", network=d["agent"]["network"][:-len("_value")], gamma=0.99,
                      use_standardization=True, lr_decay=True)
    return d


# ---- continuous off-policy family: jorldy/config/{ddpg,td3,sac}/{cartpole,pendulum,mujoco}.py --------------------------------
_TRAIN_MUJOCO = dict(training=True, load_path=None, run_step=1000000, print_period=10000, save_period=100000, eval_iteration=10)
_AC_ENVS = {"ddpg": ("cartpole", "pendulum", "mujoco"), "td3": ("cartpole", "mujoco"), "sac": ("cartpole", "pendulum", "mujoco")}


def _ac_config(agent, env):
    env_d = {"cartpole": dict(name="cartpole", action_type="continuous", render=False), "pendulum": dict(name="pendulum", render=False),
             "mujoco": dict(render=False)}[env]
    mj = env == "mujoco"
    if agent == "ddpg":
        a = dict(name="ddpg", actor="deterministic_policy", critic="continuous_q_network", gamma=0.99, buffer_size=50000,
                 batch_size=128, start_train_step=1000 if mj else 2000, tau=1e-3, lr_decay=True, mu=0, theta=1e-3, sigma=2e-3)
        opt = dict(actor="adam", critic="adam", actor_lr=5e-4, critic_lr=1e-3)
        tr = dict(_TRAIN_MUJOCO, distributed_batch_size=256, update_period=1, num_workers=8) if mj else \
            dict(_TRAIN_SMALL, eval_iteration=10, update_period=1, num_workers=8)
        if env == "pendulum":
            tr = dict(_TRAIN_SMALL, eval_iteration=10, distributed_batch_size=128, update_period=1, num_workers=8)
    elif agent == "td3":
        a = dict(name="td3", actor="deterministic_policy", critic="continuous_q_network")
        if mj:
            a.update(hidden_size=512, gamma=0.99, buffer_size=1000000, batch_size=128, start_train_step=25000,
                     initial_random_step=25000, tau=5e-3, update_delay=2, action_noise_std=0.1, target_noise_std=0.2,
                     target_noise_clip=0.5, lr_decay=True)
            opt = dict(actor="adam", critic="adam", actor_lr=3e-4, critic_lr=3e-4)
            tr = dict(_TRAIN_MUJOCO, distributed_batch_size=256, update_period=1, num_workers=8)
        else:       # td3/cartpole.py spells two keys differently from the constructor (actor_period, act_noise_std): kept as shipped
            a.update(gamma=0.99, buffer_size=50000, batch_size=128, start_train_step=1000, initial_random_step=0, tau=1e-3,
                     actor_period=2, act_noise_std=0.1, target_noise_std=0.2, target_noise_clip=0.5, lr_decay=True)
            opt = dict(actor="adam", critic="adam", actor_lr=1e-3, critic_lr=1e-3)
            tr = dict(_TRAIN_SMALL, eval_iteration=10, update_period=1, num_workers=8)
    else:
        a = dict(name="sac", actor="continuous_policy", critic="continuous_q_network", use_dynamic_alpha=True, gamma=0.99, tau=5e-3,
                 buffer_size=50000, batch_size=256 if mj else 64, start_train_step=25000 if mj else 5000, static_log_alpha=-2.0,
                 lr_decay=True)
        if env == "cartpole":
            a.update(target_update_period=500)
            a = {k: a[k] for k in ("name", "actor", "critic", "use_dynamic_alpha", "gamma", "tau", "buffer_size", "batch_size",
                                   "start_train_step", "static_log_alpha", "target_update_period", "lr_decay")}
        opt = dict(actor="adam", critic="adam", alpha="adam", actor_lr=5e-4, critic_lr=1e-3, alpha_lr=3e-4)
        if env == "cartpole":
            opt.update(actor_lr=1.5e-4, critic_lr=3e-4, alpha_lr=1e-5)
        tr = dict(_TRAIN_MUJOCO, record=False, record_period=500000, update_period=128, num_workers=16) if mj else \
            dict(_TRAIN_SMALL, eval_iteration=10, update_period=32, num_workers=8)
    return dict(env=env_d, agent=a, optim=opt, train=tr)


def _sac_discrete_config(env):
    """Discrete-action SAC (agent name "sac", actor "discrete_policy").  These follow the SAC-Discrete paper
    (Christodoulou 2019, arXiv:1910.07207), not a reference config file; a JORLDY config directory on sys.path takes
    precedence.  cartpole: config.sac.cartpole with the discrete actor and critic.  atari names no game: runs pass
    --env.name."""
    if env == "cartpole":
        d = _ac_config("sac", "cartpole")
        d["env"].update(action_type="discrete")
        d["agent"].update(actor="discrete_policy", critic="discrete_q_network")
        return d
    a = dict(name="sac", actor="discrete_policy", critic="discrete_q_network", head="cnn", use_dynamic_alpha=True, gamma=0.99,
             tau=5e-3, buffer_size=1000000, batch_size=64, start_train_step=20000)
    return dict(env=dict(_ATARI_ENV), agent=a,
                optim=dict(actor="adam", critic="adam", alpha="adam", actor_lr=3e-4, critic_lr=3e-4, alpha_lr=3e-4),
                train=dict(_TRAIN_ATARI, update_period=4, num_workers=16))


# MPO (arXiv:1806.06920): this project's choices, not a reference config file.  The agent keys are shared by every env
# (V-MPO's constructor defaults for the multipliers); buffer_size / start_train_step and the train dict are SAC's for
# the same env (mountaincar: cartpole's replay keys and the value agents' _TRAIN_SMALL row).
_MPO_KEYS = dict(name="mpo", hidden_size=512, gamma=0.99, n_step=8, batch_size=64, critic_loss_type="retrace", num_sample=30,
                 target_update_period=100, clip_grad_norm=1.0, min_eta=1e-8, min_alpha_mu=1e-8, min_alpha_sigma=1e-8,
                 eps_eta=0.01, eps_alpha_mu=0.01, eps_alpha_sigma=5e-5, eta=1.0, alpha_mu=1.0, alpha_sigma=1.0, lr_decay=True)
_MPO_ENVS = ("cartpole", "mountaincar", "pendulum", "mujoco")


def _mpo_config(env):
    """MPO: discrete_policy / discrete_q_network on cartpole and mountaincar, continuous_policy / continuous_q_network on
    pendulum and mujoco; one Adam setting (lr 3e-4) for the actor, the critic and the multipliers.  These are this
    project's choices; a JORLDY config directory on sys.path takes precedence."""
    sac = _ac_config("sac", "cartpole" if env == "mountaincar" else env)
    a = dict(_MPO_KEYS, buffer_size=sac["agent"]["buffer_size"], start_train_step=sac["agent"]["start_train_step"])
    if env in ("cartpole", "mountaincar"):
        a.update(actor="discrete_policy", critic="discrete_q_network")
    else:
        a.update(actor="continuous_policy", critic="continuous_q_network")
    if env == "cartpole":
        env_d, tr = dict(name="cartpole", action_type="discrete", render=False), sac["train"]
    elif env == "mountaincar":
        env_d, tr = dict(name="mountain_car", render=False), dict(_TRAIN_SMALL, eval_iteration=10, update_period=32, num_workers=8)
    else:
        env_d, tr = sac["env"], sac["train"]
    return dict(env=env_d, agent=a, optim=dict(name="adam", lr=3e-4), train=tr)


# MuZero (arXiv:1911.08265): this project's choices, not a reference config file; a JORLDY config directory on sys.path
# takes precedence.  gamma, the unroll, the n-step return, the simulation count, the Dirichlet noise, PER alpha / beta
# 1.0 and the value loss weight 0.25 are the paper's; the supports cover h(max |target|) of both envs (|z| <= 1 / (1 -
# gamma) = 333 for rewards of magnitude <= 1, h(333) = 17.6 <= 20); the temperature steps sit at half and three quarters
# of the run's learns (one per update_period steps).
_MUZERO_KEYS = dict(name="muzero", hidden_size=128, latent_size=64, gamma=0.997, num_simulation=50, num_unroll=5,
                    td_steps=10, value_support=20, reward_support=1, value_loss_coef=0.25, alpha=1.0, beta=1.0,
                    uniform_sample_prob=1e-3, batch_size=128, buffer_size=100000, start_train_step=2000,
                    clip_grad_norm=5.0, root_dirichlet_alpha=0.25, root_exploration_fraction=0.25,
                    temperature_learns=(3125, 4688), lr_decay=True)
_MUZERO_ENVS = ("cartpole", "mountaincar", "atari", "tictactoe", "tictactoe_selfplay")
# Atari frames (CNN representation over 4 frames + 4 action planes).  The paper's: gamma 0.997, K = 5, n = 10, S = 50,
# the Dirichlet noise, PER alpha = beta = 1, the value loss weight 0.25, batch 1024.  This project's choices: Adam at
# 3e-4 (the paper: SGD with momentum), the 1 M-window replay and 100 k warm-up steps of the other Atari replay configs,
# hidden 512 / latent 256 flat-latent dynamics and prediction MLPs (the paper: a ResNet on 6x6 spatial latents), the
# supports 20 / 1 of the flat configs, which cover the sign-clipped rewards (the paper's 300 / 300 are for unclipped
# rewards), 32 envs with one learn every 8 rounds of env steps (3.75 M learns in the 30 M-step run), and the temperature
# steps at half and three quarters of those learns.
_MUZERO_ATARI_KEYS = dict(_MUZERO_KEYS, head="cnn", hidden_size=512, latent_size=256, batch_size=1024,
                          buffer_size=1000000, start_train_step=100000, temperature_learns=(1875000, 2812500))


def _muzero_config(env):
    if env == "atari":
        return dict(env=dict(_ATARI_ENV), agent=dict(_MUZERO_ATARI_KEYS), optim=dict(name="adam", lr=3e-4),
                    train=dict(_TRAIN_ATARI, update_period=8, num_workers=32))
    if env == "tictactoe":
        # TicTacToe (this project's choices): CartPole's settings with the paper's gamma 1 for board games, td_steps 5 (the
        # longest game), so every value target is the game's outcome in {-1, 0, 1}, and value_support 1, which covers
        # h(1) = 0.415 like the reward support
        d = _muzero_config("cartpole")
        d["env"] = dict(name="tictactoe", render=False)
        d["agent"].update(gamma=1.0, td_steps=5, value_support=1)
        return d
    if env == "tictactoe_selfplay":
        # two-player self-play (the paper's training for board games): the agent plays both sides and its search and
        # value targets alternate sides; td_steps 9, the longest game in plies, so with gamma 1 every value target is
        # the game's outcome for the side to move
        d = _muzero_config("tictactoe")
        d["env"]["opponent"] = "self"
        d["agent"].update(two_player=True, td_steps=9)
        return d
    env_d = dict(name="cartpole", action_type="discrete", render=False) if env == "cartpole" else \
        dict(name="mountain_car", render=False)
    return dict(env=env_d, agent=dict(_MUZERO_KEYS), optim=dict(name="adam", lr=3e-4),
                train=dict(_TRAIN_SMALL, eval_iteration=10, update_period=16, num_workers=8))


def available():
    out = []
    for ag, envs in _AC_ENVS.items():
        out += [f"config.{ag}.{e}" for e in envs]
    out += [f"config.sac_discrete.{e}" for e in ("cartpole", "atari")]
    for ag in list(_VALUE_AGENTS) + ["ape_x", "r2d2"]:
        out += [f"config.{ag}.{e}" for e in ("cartpole", "mountaincar", "atari")]
    out += [f"config.ppo.{e}" for e in ("cartpole", "mountaincar", "pendulum", "mujoco", "atari")]
    out += [f"config.vmpo.{e}" for e in _VMPO_ENVS]
    out += [f"config.icm_ppo.{e}" for e in _ICM_PPO_ENVS]
    out += [f"config.rnd_ppo.{e}" for e in _RND_PPO_ENVS]
    out += [f"config.mpo.{e}" for e in _MPO_ENVS]
    out += [f"config.reinforce.{e}" for e in _REINFORCE_ENVS]
    out += [f"config.muzero.{e}" for e in _MUZERO_ENVS]
    return out


def load(config_path):
    parts = config_path.split(".")
    if len(parts) != 3 or parts[0] != "config":
        raise ImportError(f"no config '{config_path}' (built-ins: {available()})")
    _, agent, env = parts
    if agent in _VALUE_AGENTS and env in ("cartpole", "mountaincar", "atari"):
        d = _value_config(agent, env)
    elif agent == "ape_x" and env in ("cartpole", "mountaincar", "atari"):
        d = _ape_x_config(env)
    elif agent == "r2d2" and env in ("cartpole", "mountaincar", "atari"):
        d = _r2d2_config(env)
    elif agent == "ppo" and env in ("cartpole", "mountaincar", "pendulum", "mujoco", "atari"):
        d = _ppo_config(env)
    elif agent == "vmpo" and env in _VMPO_ENVS:
        d = _vmpo_config(env)
    elif agent == "icm_ppo" and env in _ICM_PPO_ENVS:
        d = _icm_ppo_config(env)
    elif agent == "rnd_ppo" and env in _RND_PPO_ENVS:
        d = _rnd_ppo_config(env)
    elif agent == "mpo" and env in _MPO_ENVS:
        d = _mpo_config(env)
    elif agent == "reinforce" and env in _REINFORCE_ENVS:
        d = _reinforce_config(env)
    elif agent == "muzero" and env in _MUZERO_ENVS:
        d = _muzero_config(env)
    elif agent in _AC_ENVS and env in _AC_ENVS[agent]:
        d = _ac_config(agent, env)
    elif agent == "sac_discrete" and env in ("cartpole", "atari"):
        d = _sac_discrete_config(env)
    else:
        raise ImportError(f"no config '{config_path}' (built-ins: {available()})")
    return SimpleNamespace(**d)
