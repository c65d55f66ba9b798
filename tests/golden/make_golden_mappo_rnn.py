"""Generate tests/golden/mappo_rnn_buffer.npz by running the UNMODIFIED reference's MARL_OnPolicyBuffer_RNN
(xuance/common/memory_tools_marl.py:273-515, agi-brain/xuance v1.4.4 @ 4f0b05b) through tests/mappo_rnn_refs.py's scenario.

Run in the build container only (needs /root/reference):   python tests/golden/make_golden_mappo_rnn.py

For use_gae in {True, False} x ValueNorm {off, on}: the staging (episode_data) and the ring (data) after every op, the
ValueNorm state at each finish, and sample(SAMPLE).  Non-GAE with a ValueNorm raises a shape-mismatch error in the
reference (memory_tools_marl.py:484-489); the fixture records the message."""
import os

import numpy as np
import torch

from make_golden import ENV, HERE  # noqa: E402  (imports the reference and sets up sys.path)
from gymnasium.spaces import Box, Discrete  # noqa: E402
from xuance.common import AgentGrouping  # noqa: E402
from xuance.common.memory_tools_marl import MARL_OnPolicyBuffer_RNN  # noqa: E402
from xuance.torch.utils import ValueNorm  # noqa: E402
from mappo_rnn_refs import scenario, KEYS, N_ENVS, T_MAX, SLOTS, OBS, STATE, A, SAMPLE  # noqa: E402


def _flat(prefix, d, out):
    for k, v in d.items():
        if isinstance(v, dict):
            _flat(prefix + k + "/", v, out)
        else:
            out[prefix + k] = np.asarray(v).copy()


def main():
    out = {"env": ENV}
    grouping = AgentGrouping.shared(KEYS)
    for use_gae in (True, False):
        for vn_on in (False, True):
            case = f"gae{int(use_gae)}_vn{int(vn_on)}/"
            buf = MARL_OnPolicyBuffer_RNN(KEYS, state_space=Box(-1, 1, (STATE,)),
                                          obs_space={k: Box(-1, 1, (OBS,)) for k in KEYS},
                                          act_space={k: Discrete(A) for k in KEYS}, n_envs=N_ENVS, buffer_size=SLOTS,
                                          max_episode_steps=T_MAX, use_gae=use_gae, use_advnorm=True, gamma=0.99,
                                          gae_lam=0.95, use_actions_mask=True,
                                          avail_actions_shape={k: (A,) for k in KEYS})
            vn = {"shared": ValueNorm(1)} if vn_on else None
            if vn_on:       # a non-trivial state before the first finish
                vn["shared"].update(torch.tensor(np.linspace(-2, 5, 12, dtype=np.float32)[:, None]))
            for j, op in enumerate(scenario()):
                if op[0] == "store":
                    buf.store(**op[1])
                elif op[0] == "vn_update":
                    if vn_on:
                        vn["shared"].update(torch.from_numpy(op[1]))
                else:
                    _, e, i_step, vnext = op
                    if vn_on:
                        out[case + f"op{j}/vn"] = np.array([vn["shared"].running_mean.item(),
                                                            vn["shared"].running_mean_sq.item(),
                                                            vn["shared"].debiasing_term.item()], np.float32)
                    try:
                        buf.finish_path(i_env=e, i_step=i_step, agent_grouping=grouping, value_next=vnext,
                                        value_normalizer=vn)
                    except ValueError as exc:     # the reference's non-GAE branch with a ValueNorm (DESIGN §4)
                        out[case + "raises"] = np.array(str(exc))
                        break
                    _flat(case + f"op{j}/staging/", buf.episode_data, out)
            if case + "raises" in out:
                continue
            _flat(case + "data/", buf.data, out)
            _flat(case + "staging/", buf.episode_data, out)
            out[case + "ptr_size"] = np.array([buf.ptr, buf.size])
            s = buf.sample(np.array(SAMPLE))
            _flat(case + "sample/", {k: v for k, v in s.items() if k not in ("batch_size", "sequence_length")}, out)
            out[case + "sample_meta"] = np.array([s["batch_size"], s["sequence_length"]])
    np.savez_compressed(os.path.join(HERE, "mappo_rnn_buffer.npz"), **out)


if __name__ == "__main__":
    main()
