from .learner import Learner
from .ppo_learner import PPO_Learner, A2C_Learner, PG_Learner
from .dqn_learner import DQN_Learner, PerDQN_Learner, DDQN_Learner, DuelDQN_Learner
from .dist_dqn_learner import C51_Learner, QRDQN_Learner
from .sac_learner import SAC_Learner
from .sacdis_learner import SACDIS_Learner
from .ddpg_learner import DDPG_Learner, TD3_Learner
from .qmix_learner import QMIX_Learner
from .wqmix_learner import WQMIX_Learner
from .dcg_learner import DCG_Learner
from .qtran_learner import QTRAN_Learner
from .iql_learner import IQL_Learner
from .mappo_learner import MAPPO_Learner
from .vdac_learner import VDAC_Learner, IAC_Learner
from .coma_learner import COMA_Learner
from .ppg_learner import PPG_Learner
from .npg_learner import NPG_Learner
from .drqn_learner import DRQN_Learner

REGISTRY_Learners = {"PPO_Learner": PPO_Learner, "PPOCLIP_Learner": PPO_Learner, "DQN_Learner": DQN_Learner,
                     "PerDQN_Learner": PerDQN_Learner, "DDQN_Learner": DDQN_Learner, "A2C_Learner": A2C_Learner,
                     "PG_Learner": PG_Learner, "DuelDQN_Learner": DuelDQN_Learner,
                     "C51_Learner": C51_Learner, "QRDQN_Learner": QRDQN_Learner,
                     "SAC_Learner": SAC_Learner, "SACDIS_Learner": SACDIS_Learner,
                     "DDPG_Learner": DDPG_Learner, "TD3_Learner": TD3_Learner,
                     "QMIX_Learner": QMIX_Learner,
                     "VDN_Learner": QMIX_Learner,     # vdn_learner.py: the same update with the parameter-free sum mixer
                     "MAPPO_Learner": MAPPO_Learner, "PPG_Learner": PPG_Learner, "NPG_Learner": NPG_Learner, "WQMIX_Learner": WQMIX_Learner,
                     "DCG_Learner": DCG_Learner, "QTRAN_Learner": QTRAN_Learner, "IQL_Learner": IQL_Learner,
                     "VDAC_Learner": VDAC_Learner, "IAC_Learner": IAC_Learner,
                     "DRQN_Learner": DRQN_Learner, "COMA_Learner": COMA_Learner}
