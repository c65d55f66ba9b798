from .layers import mlp_block, cnn_block, ActivationFunctions
from .outputs import (ModelOutput, RNN_State, RepresentationOutput, ActionOutput, StochasticActorOutput, TwinCriticOutput,
                      DeterministicActorOutput, CriticOutput)
from .distributions import CategoricalDistribution, DiagGaussianDistribution, ActivatedDiagGaussianDistribution
from .representations import Basic_Identical, Basic_MLP, Basic_CNN, AC_CNN_Atari, REGISTRY_Representation
from .heads import (CategoricalActorHead, GaussianActorHead, SAC_GaussianActorHead, ValueHead, QValueHead, DuelingQValueHead,
                    DeterministicActorHead, C51QValueHead, QuantileRegressionQValueHead)
from .architectures import (ActorCritic, SharedActorCritic, DeepQNetwork, DuelingDeepQNetwork, GaussianActor, SAC_GaussianActor,
                            TwinActionValueCritic, SoftActorCritic, TwinDiscreteActionValueCritic, SoftActorCriticDiscrete,
                            DeterministicActor, ActionValueCritic, DeterministicActorCritic, TwinDelayedActorCritic,
                            C51DeepQNetwork, QRDeepQNetwork, StateValueCritic, PhasicActorCritic)
from .qmix import (Basic_RNN, AgentFeatureEncoder, DiscreteActionValueCritic, QMIX_Mixer, VDN_mixer, MixingQNetwork,
                   QMIX_FF_Mixer, WeightedMixingQNetwork, IndependentMixer)
REGISTRY_Representation["Basic_RNN"] = Basic_RNN
from .mappo import CategoricalActor, CentralizedStateValueCritic, MultiAgentActorCritic
from .gru import GRUSequence, gru_sequence, Basic_RNN_K13
from .dcg import DCG_Utility, DCG_Payoff, Coordination_Graph, DeepCoordinationGraph
from .qtran import QTRAN_Base, QTRAN_Alt, QTranMixingNetwork
from .vdac import IndependentActorCritic, ValueDecompositionActorCritic
from .lstm import LSTMSequence, lstm_sequence
from .drqn import RecurrentQValueHead, DeepRecurrentQNetwork
from .coma import CounterfactualCentralizedCritic, CounterfactualMultiAgentActorCritic
