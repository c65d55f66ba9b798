from .learner import Learner
from .ppo_learner import PPO_Learner, A2C_Learner, PG_Learner
from .dqn_learner import DQN_Learner, PerDQN_Learner, DDQN_Learner, DuelDQN_Learner
from .dist_dqn_learner import C51_Learner, QRDQN_Learner

REGISTRY_Learners = {"PPO_Learner": PPO_Learner, "PPOCLIP_Learner": PPO_Learner, "DQN_Learner": DQN_Learner,
                     "PerDQN_Learner": PerDQN_Learner, "DDQN_Learner": DDQN_Learner, "A2C_Learner": A2C_Learner,
                     "PG_Learner": PG_Learner, "DuelDQN_Learner": DuelDQN_Learner,
                     "C51_Learner": C51_Learner, "QRDQN_Learner": QRDQN_Learner}
try:
    from .sac_learner import SAC_Learner
    REGISTRY_Learners["SAC_Learner"] = SAC_Learner
    from .sacdis_learner import SACDIS_Learner
    REGISTRY_Learners["SACDIS_Learner"] = SACDIS_Learner
    from .ddpg_learner import DDPG_Learner, TD3_Learner
    REGISTRY_Learners["DDPG_Learner"] = DDPG_Learner
    REGISTRY_Learners["TD3_Learner"] = TD3_Learner
except ImportError:
    pass
try:
    from .qmix_learner import QMIX_Learner
    REGISTRY_Learners["QMIX_Learner"] = QMIX_Learner
    REGISTRY_Learners["VDN_Learner"] = QMIX_Learner     # vdn_learner.py: the same update with the parameter-free sum mixer
except ImportError:
    pass
from .mappo_learner import MAPPO_Learner
REGISTRY_Learners["MAPPO_Learner"] = MAPPO_Learner
