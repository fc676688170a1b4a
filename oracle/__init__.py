"""CPU oracle for the jorldy_b200 hot path — TEST INFRASTRUCTURE, not product code.

A restatement (numpy + torch-CPU fp32) of the reference algorithms on the
rollout-collect -> buffer -> learn() path of kakaoenterprise/JORLDY, each function citing the
reference file:line it follows.  Only tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs may import it; the product package (jorldy_b200/) never does
and fails loudly when its CUDA library is missing.

Pinning status
  * learner maths (PPO / DQN family / C51 / Rainbow / Ape-X learn(), PER buffer, GAE): pinned
    against outputs of the UNMODIFIED reference classes imported in the build container
    (tests/golden/make_golden.py generated tests/golden/*.npz; tests/test_oracle_golden.py replays
    them through this package).  The reference itself ships no float golden vectors
    (SURVEY.md §8c), only bookkeeping asserts; those are re-run against the CUDA classes in
    tests/test_per_gpu.py, test_replay_gpu.py, test_dqn_gpu.py, test_ppo_gpu.py and test_ac_gpu.py.
  * collect side (act sampling, n-step assemblers, collect loops: oracle/collect.py) and the continuous off-policy
    family (DDPG / TD3 / SAC learn() and act(): oracle/actor_critic.py): pinned the same way — fixtures minted from the
    reference's own act() / interact_callback() / learn() with every random primitive replaced by an injected draw
    (tests/golden/make_golden_collect.py, make_golden_ac.py, make_golden_ac_act.py).
  * CartPole / Pendulum / MountainCar physics: gym==0.23.0 is a third-party dependency that is
    NOT vendored in the reference and is not installed (requirements.txt:2).  Its
    published equations are restated in oracle/classic_control.py; the reference's own tests for
    the envs check shapes only (jorldy/test/core/env/test_gym_env.py:5-32).  PARITY UNPINNED for
    the physics constants; pinned only for JORLDY's wrapper semantics (reward override, shapes).
"""
