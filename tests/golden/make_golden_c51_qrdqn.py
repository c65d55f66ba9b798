"""Generate tests/golden/c51_qrdqn_update.npz by running the UNMODIFIED reference (agi-brain/xuance v1.4.4 @ 4f0b05b).

Run in the build container only (needs the reference checkout):   python tests/golden/make_golden_c51_qrdqn.py
Reuses make_golden.py's reference import (read-only, with the oracle/ref_stubs import stubs) and environment-of-record
string; writes only this one fixture.

Four updates each of C51_Learner (c51_learner.py:27-81, 51 atoms on [-10, 10]) and QRDQN_Learner (qrdqn_learner.py:29-77,
20 quantiles) on the reference's own C51DeepQNetwork / QRDeepQNetwork over a Basic_MLP encoder (6-d observations, 32
units, head [32], 3 actions), sync_frequency 2 so that the hard target copy happens inside the fixture, batch 40 with
terminal rows and rewards that clamp Tz at both v_min and v_max; once with use_grad_clip off (``<algo>/clip0/``) and
once on with a binding norm (``<algo>/clip1/``).  Per update: the info dict and the full state_dict (C51's includes
``supports``: the model is built on the CPU)."""
import os

import numpy as np
import torch

from make_golden import ENV, HERE, _learner_cfg  # noqa: E402  (imports the reference and sets up sys.path)
from gymnasium.spaces import Discrete  # noqa: E402
from xuance.common import BaseCallback  # noqa: E402
from xuance.torch.rl_models.representations.mlp import Basic_MLP  # noqa: E402
from xuance.torch.rl_models.architectures import C51DeepQNetwork, QRDeepQNetwork  # noqa: E402
from xuance.torch.learners import C51_Learner, QRDQN_Learner  # noqa: E402
from dist_refs import (OBS, HIDDEN, N_ACT, ATOMS, QUANTILES, V_MIN, V_MAX, GAMMA, LR, SYNC, N_UPDATES,  # noqa: E402
                       CLIP_NORM, fixture_batch, fixture_state_dict)

KEYS = ["Qloss", "learning_rate"]


def build_reference_model(algo):
    init, act = torch.nn.init.orthogonal_, torch.nn.ReLU
    rep = Basic_MLP((OBS,), [HIDDEN], None, init, act, 'cpu')
    if algo == "c51":
        model = C51DeepQNetwork(rep, [HIDDEN], Discrete(N_ACT), ATOMS, V_MIN, V_MAX, None, init, act, 'cpu')
    else:
        model = QRDeepQNetwork(rep, [HIDDEN], Discrete(N_ACT), QUANTILES, None, init, act, 'cpu')
    model.load_state_dict(fixture_state_dict(model.state_dict()))
    return model


def learner_cfg(clip):
    return _learner_cfg(learning_rate=LR, gamma=GAMMA, sync_frequency=SYNC, use_grad_clip=clip, grad_clip_norm=CLIP_NORM,
                        end_factor_lr_decay=0.5, parallels=4, running_steps=64, start_training=0, training_frequency=1)


def golden(out, algo, clip):
    pre = f"{algo}/clip{int(clip)}/"
    model = build_reference_model(algo)
    lrn = (C51_Learner if algo == "c51" else QRDQN_Learner)(learner_cfg(clip), model, BaseCallback())
    out[pre + "total_iters"] = lrn.total_iters
    for k, v in model.state_dict().items():
        out[f"{pre}init/{k}"] = v.detach().numpy().copy()
    rng = np.random.default_rng(80 + 2 * (algo == "qrdqn") + clip)
    infos = []
    for it in range(N_UPDATES):
        info = lrn.update(**fixture_batch(rng))
        infos.append([float(info[k]) for k in KEYS])
        for k, v in model.state_dict().items():
            out[f"{pre}it{it}/{k}"] = v.detach().numpy().copy()
    out[pre + "infos"] = np.array(infos, np.float64)


if __name__ == "__main__":
    out = {"env": ENV}
    for algo in ("c51", "qrdqn"):
        for clip in (False, True):
            golden(out, algo, clip)
    path = os.path.join(HERE, "c51_qrdqn_update.npz")
    np.savez_compressed(path, **out)
    print("c51_qrdqn_update.npz", os.path.getsize(path))
