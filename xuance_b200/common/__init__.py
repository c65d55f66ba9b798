from .spaces import Space, Box, Discrete, space2shape, combined_shape, is_discrete
from .memory_tools import (Buffer, DummyOnPolicyBuffer, DummyOnPolicyBuffer_Atari, DummyOffPolicyBuffer,
                           DummyOffPolicyBuffer_Atari, PerOffPolicyBuffer, PreparedObs,
                           RecurrentOffPolicyBuffer)
from .callback import BaseCallback
from .agent_grouping import AgentGrouping
from .memory_tools_marl import MARL_OffPolicyBuffer_RNN, MARL_OnPolicyBuffer, MARL_OnPolicyBuffer_RNN
