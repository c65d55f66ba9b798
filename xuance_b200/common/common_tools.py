"""Config loading (reference: xuance/common/common_tools.py:10-146): ``basic.yaml`` (+) ``configs/<algo>/<env>.yaml``
(+) parser args -> SimpleNamespace.  Same merge rule (recursive dict update, later wins)."""
import os
from copy import deepcopy
from types import SimpleNamespace as SN

import yaml

EPS = 1e-8
_CONFIG_ROOT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "configs")


def recursive_dict_update(basic_dict, target_dict):
    out = deepcopy(basic_dict)
    for k, v in target_dict.items():
        out[k] = recursive_dict_update(out.get(k, {}), v) if isinstance(v, dict) else v
    return out


def load_yaml(file_dir):
    with open(file_dir, "r") as f:
        return yaml.load(f, Loader=yaml.FullLoader)


def get_arguments(algo, env, env_id=None, config_path=None, parser_args=None):
    """``algo`` e.g. 'ppo', ``env`` e.g. 'atari' / 'classic_control', ``env_id`` e.g. 'CartPole-v1'."""
    cfg = load_yaml(os.path.join(_CONFIG_ROOT, "basic.yaml"))
    if config_path is None:
        # the third candidate is the reference's own layout, configs/<algo>/<env>/<env_id>.yaml
        cands = [os.path.join(_CONFIG_ROOT, algo, f"{env_id}.yaml"), os.path.join(_CONFIG_ROOT, algo, f"{env}.yaml"),
                 os.path.join(_CONFIG_ROOT, algo, env, f"{env_id}.yaml")]
        found = [c for c in cands if os.path.exists(c)]
        if not found:
            raise AttributeError(f"no config for algo={algo} env={env} env_id={env_id} under {_CONFIG_ROOT}")
        config_path = found[0]
    cfg = recursive_dict_update(cfg, load_yaml(config_path))
    if parser_args is not None:
        cfg = recursive_dict_update(cfg, parser_args.__dict__ if hasattr(parser_args, "__dict__") else dict(parser_args))
    return SN(**cfg)
