from .agent import Agent, set_seed, set_device
from .on_policy import OnPolicyAgent
from .off_policy import OffPolicyAgent
from .ppo_agent import PPO_Agent
from .dqn_agent import DQN_Agent, PerDQN_Agent, DuelDQN_Agent
from .dist_dqn_agent import C51_Agent, QRDQN_Agent
from .ppg_agent import PPG_Agent
from .npg_agent import NPG_Agent
# DRQN_Agent is constructed directly, DRQN_Agent(config, envs): adding it to REGISTRY_Agents (and so to get_runner) is a
# separate change, because the registry's keys are pinned by the C51 / QR-DQN tests
from .drqn_agent import DRQN_Agent

REGISTRY_Agents = {"PPO": PPO_Agent, "PPO_Clip": PPO_Agent, "DQN": DQN_Agent, "PerDQN": PerDQN_Agent, "DuelDQN": DuelDQN_Agent,
                   "C51DQN": C51_Agent, "QRDQN": QRDQN_Agent, "PPG": PPG_Agent,
                   "NPG": NPG_Agent}
try:
    from .sac_agent import SAC_Agent
    REGISTRY_Agents["SAC"] = SAC_Agent
    from .ddpg_agent import DDPG_Agent, TD3_Agent
    REGISTRY_Agents["DDPG"] = DDPG_Agent
    REGISTRY_Agents["TD3"] = TD3_Agent
except ImportError:
    pass
from .marl import MARLAgents, OffPolicyMARLAgents, QMIX_Agents, VDN_Agents
from .wqmix_agents import WQMIX_Agents
REGISTRY_Agents["QMIX"] = QMIX_Agents
REGISTRY_Agents["VDN"] = VDN_Agents
REGISTRY_Agents["OWQMIX"] = WQMIX_Agents
REGISTRY_Agents["CWQMIX"] = WQMIX_Agents
from .dcg_agents import DCG_Agents
REGISTRY_Agents["DCG"] = DCG_Agents
REGISTRY_Agents["DCG_S"] = DCG_Agents
from .qtran_agents import QTRAN_Agents
REGISTRY_Agents["QTRAN_base"] = QTRAN_Agents
REGISTRY_Agents["QTRAN_alt"] = QTRAN_Agents
from .iql_agents import IQL_Agents
REGISTRY_Agents["IQL"] = IQL_Agents
from .mappo_agents import OnPolicyMARLAgents, MAPPO_Agents, IPPO_Agents
REGISTRY_Agents["MAPPO"] = MAPPO_Agents
REGISTRY_Agents["IPPO"] = IPPO_Agents
from .vdac_agents import VDAC_Agents, IAC_Agents
REGISTRY_Agents["VDAC"] = VDAC_Agents
REGISTRY_Agents["IAC"] = IAC_Agents
from .coma_agents import COMA_Agents
REGISTRY_Agents["COMA"] = COMA_Agents
