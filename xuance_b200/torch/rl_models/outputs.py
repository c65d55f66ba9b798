"""Output records (reference: xuance/torch/rl_models/modules/outputs.py:8-80) - same field names."""
from dataclasses import dataclass, field
from typing import Any, Optional


@dataclass
class RNN_State:
    hidden_states: Any = None
    cell_states: Any = None


@dataclass
class RepresentationOutput:
    embeddings: Any
    rnn_states: Any = None
    aux: dict = field(default_factory=dict)


@dataclass
class StochasticActorOutput:
    representations: Any
    distributions: Any = None


@dataclass
class DeterministicActorOutput:
    representations: Any
    actions: Any = None


@dataclass
class CriticOutput:
    representations: Any
    values: Any = None


@dataclass
class TwinCriticOutput:
    representations_1: Any
    representations_2: Any
    values_1: Any
    values_2: Any


@dataclass
class ModelOutput:
    actions: Any = None
    distributions: Any = None
    values: Any = None
    rep_out: Any = None
    actor_rep_out: Any = None
    critic_rep_out: Any = None


@dataclass
class ActionOutput:
    env_actions: Any
    policy_actions: Any = None
    distributions: Any = None
    log_probs: Any = None
    values: Any = None
    rnn_hidden: Any = None
