"""Policy-only networks of the continuous off-policy family (jorldy/core/network/policy.py).

`DeterministicPolicy` (policy.py:8-20: head -> l -> tanh(pi), used by DDPG / TD3) and `ContinuousPolicy`
(policy.py:38-56: head -> l -> {mu clamped to +-5, std = exp(tanh(log_std))}, used by SAC) and `DiscretePolicy`
(head -> l -> softmax logits, used by the discrete-action SAC) are the trunk +
narrow-heads shape of policy_value.py without the value head; forward_raw returns the PRE-activation head
outputs, the activations live in csrc/actor_critic.cu."""
from .policy_value import _PolicyValue


class DeterministicPolicy(_PolicyValue):
    def _out_heads(self, D_out):
        return [("pi", D_out, "tanh")]


class ContinuousPolicy(_PolicyValue):
    def _out_heads(self, D_out):
        return [("mu", D_out, "linear"), ("log_std", D_out, "tanh")]


class DiscretePolicy(_PolicyValue):
    """The reference's `discrete_policy`: head -> l -> pi.  forward_raw returns the logits; the softmax lives in the
    discrete SAC kernels (csrc/actor_critic.cu jb_sacd_*)."""

    def _out_heads(self, D_out):
        return [("pi", D_out, "policy")]
