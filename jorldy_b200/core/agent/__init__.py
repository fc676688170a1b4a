"""Agent factory with the reference's registry keys (jorldy/core/agent/__init__.py:32-42)."""
from collections import OrderedDict

from .ppo import PPO
from .dqn import DQN, Double, Dueling, Multistep, PER, Noisy, C51, Rainbow, ApeX
from .ddpg import DDPG, TD3, SAC
from .quantile import IQN, QRDQN
from .munchausen import MDQN, MIQN
from .rainbow_iqn import RainbowIQN
from .r2d2 import R2D2
from .vmpo import VMPO
from .icm_ppo import ICM_PPO
from .mpo import MPO
from .rnd_ppo import RND_PPO
from .reinforce import REINFORCE

agent_dict = OrderedDict(sorted(dict(ape_x=ApeX, c51=C51, ddpg=DDPG, double=Double, dqn=DQN, dueling=Dueling, icm_ppo=ICM_PPO, iqn=IQN,
                                     m_dqn=MDQN, m_iqn=MIQN, mpo=MPO, multistep=Multistep, noisy=Noisy, per=PER, ppo=PPO, qrdqn=QRDQN, r2d2=R2D2,
                                     rainbow=Rainbow, rainbow_iqn=RainbowIQN, reinforce=REINFORCE, rnd_ppo=RND_PPO, sac=SAC, td3=TD3,
                                     vmpo=VMPO).items()))


def register(name, cls):
    agent_dict[name] = cls


class Agent:
    def __new__(cls, name, *args, **kwargs):
        if type(name) != str:
            print("### name variable must be string! ###")
            raise Exception
        name = name.lower()
        if name not in agent_dict.keys():
            print(f"### can use only follows {[opt for opt in agent_dict.keys()]}")
            raise Exception
        return agent_dict[name](*args, **kwargs)
