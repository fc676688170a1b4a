"""Env factory with the reference's registry keys (jorldy/core/env/__init__.py:41-64)."""
from collections import OrderedDict

from .classic import Cartpole, Pendulum, MountainCar
from .frames import SyntheticAtari, _ACTIONS
from .synth import SyntheticControl, _DIMS
from .tictactoe import TicTacToe

env_dict = OrderedDict(cartpole=Cartpole, mountain_car=MountainCar, pendulum=Pendulum, synthetic_atari=SyntheticAtari,
                       tictactoe=TicTacToe)
for _game in _ACTIONS:            # atari.py registers one class per game (Breakout, Pong, ...)
    env_dict[_game] = (lambda g: (lambda **kw: SyntheticAtari(name=g, **kw)))(_game)


for _task in _DIMS:              # mujoco.py registers one class per task (Hopper, HalfCheetah, ...)
    env_dict[_task] = (lambda g: (lambda **kw: SyntheticControl(name=g, **kw)))(_task)


def register(name, cls):
    env_dict[name] = cls


class Env:
    def __new__(cls, name, *args, **kwargs):
        if type(name) != str:
            print("### name variable must be string! ###")
            raise Exception
        name = name.lower()
        if name not in env_dict.keys():
            print(f"### can use only follows {[opt for opt in env_dict.keys()]}")
            raise Exception
        return env_dict[name](*args, **kwargs)
