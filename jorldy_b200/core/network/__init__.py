"""Network factory with the reference's registry keys (jorldy/core/network/__init__.py:30-40:
snake_case(ClassName))."""
from collections import OrderedDict

from .policy_value import DiscretePolicyValue, ContinuousPolicyValue, DiscreteQ_Network
from .dueling import Dueling
from .iqn import IQN
from .noisy import Noisy, Rainbow
from .policy import ContinuousPolicy, DeterministicPolicy, DiscretePolicy
from .q_network import ContinuousQ_Network
from .r2d2 import R2D2
from .rainbow_iqn import RainbowIQN

network_dict = OrderedDict(
    continuous_policy=ContinuousPolicy,
    continuous_policy_value=ContinuousPolicyValue,
    continuous_q_network=ContinuousQ_Network,
    deterministic_policy=DeterministicPolicy,
    discrete_policy=DiscretePolicy,
    discrete_policy_value=DiscretePolicyValue,
    discrete_q_network=DiscreteQ_Network,
    dueling=Dueling,
    iqn=IQN,
    noisy=Noisy,
    r2d2=R2D2,
    rainbow=Rainbow,
    rainbow_iqn=RainbowIQN,
)


def register(name, cls):
    network_dict[name] = cls


class Network:
    def __new__(cls, name, *args, **kwargs):
        if type(name) != str:
            print("### name variable must be string! ###")
            raise Exception
        name = name.lower()
        if name not in network_dict.keys():
            print(f"### can use only follows {[opt for opt in network_dict.keys()]}")
            raise Exception
        return network_dict[name](*args, **kwargs)
