"""The recurrent MAPPO buffer scenario shared by tests/golden/make_golden_mappo_rnn.py (run on the reference's
MARL_OnPolicyBuffer_RNN) and the GPU tests (run on the device buffer): 2 envs x 3 agents, T_max = 6, 4 episode slots,
global state and action masks.  env 0 finishes at episode step 3 (terminal) and again at 2 (terminal), so its second
episode's padded tail still holds the first one's data; env 1 is truncated at T_max = 6 (bootstrapped) and again at 2.
The ValueNorm is updated between finishes, so each finish_path denormalises with a different state."""
import numpy as np

N_ENVS, N_AGENTS, T_MAX, SLOTS, OBS, STATE, A = 2, 3, 6, 4, 5, 7, 4
KEYS = [f"agent_{i}" for i in range(N_AGENTS)]
ENDS = {0: [(3, True), (2, True)], 1: [(6, False), (2, False)]}     # (episode length, terminal) per env
G = 8                                                                # vector steps
SAMPLE = [2, 0, 3, 1]


def scenario(seed=0):
    """List of ops: ("store", step_data) / ("finish", i_env, i_step, value_next) / ("vn_update", x [k, 1])."""
    rng = np.random.default_rng(seed)
    ops, ep_step, ends = [], [0, 0], {e: list(v) for e, v in ENDS.items()}
    for g in range(G):
        ep_step = [s + 1 for s in ep_step]
        f = lambda *a: {k: rng.normal(*a, N_ENVS).astype(np.float32) for k in KEYS}
        done = {e: bool(ends[e]) and ep_step[e] == ends[e][0][0] for e in range(N_ENVS)}
        term = {k: np.array([done[e] and ends[e][0][1] for e in range(N_ENVS)]) for k in KEYS}
        avail = {k: (rng.random((N_ENVS, A)) > 0.3) for k in KEYS}
        acts = {k: np.array([np.flatnonzero(avail[k][e])[0] if avail[k][e].any() else 0 for e in range(N_ENVS)],
                            np.float32) for k in KEYS}
        for k in KEYS:
            avail[k][np.arange(N_ENVS), acts[k].astype(int)] = True
        ops.append(("store", {
            'obs': {k: rng.normal(size=(N_ENVS, OBS)).astype(np.float32) for k in KEYS}, 'actions': acts,
            'log_pi_old': f(-1.0, 0.3), 'rewards': f(0.5, 1.0), 'values': f(0.0, 1.0), 'terminals': term,
            'agent_mask': {k: rng.random(N_ENVS) > 0.2 for k in KEYS}, 'avail_actions': avail,
            'state': rng.normal(size=(N_ENVS, STATE)).astype(np.float32),
            'episode_steps': np.array([s - 1 for s in ep_step])}))
        if g == 4:
            ops.append(("vn_update", rng.normal(2.0, 3.0, (16, 1)).astype(np.float32)))
        for e in range(N_ENVS):
            if done[e]:
                terminal = ends[e][0][1]
                vnext = {k: 0.0 for k in KEYS} if terminal else {k: np.float32(rng.normal()) for k in KEYS}
                ops.append(("finish", e, ep_step[e], vnext))
                ends[e].pop(0)
                ep_step[e] = 0
    return ops
