"""TEST INFRASTRUCTURE (see oracle/__init__.py).  Restatement of the reference's agent-side loops that drive the hot path,
used to prove the drop-in claim in two steps: tests/test_dropin_reference.py runs THIS function against recording fakes
and requires the call sequence the reference's ``xuance.torch.agents.core.on_policy.OnPolicyAgent.train_epochs`` produced
(recorded by tests/golden/make_reference_live.py); tests/test_gpu_dropin.py runs this function over the real
xuance_b200 buffer + learner on the GPU and requires the result of the product agent's own ``train_epochs``."""
import numpy as np


def reference_train_epochs(agent, n_epochs=1):
    """xuance/torch/agents/core/on_policy.py:182-205: ``indexes`` is created once and shuffled in place every epoch with
    NumPy's global RNG; every minibatch is ``memory.sample(indexes[start:end])`` -> ``learner.update(**samples)``; the info of
    the LAST minibatch is returned."""
    indexes = np.arange(agent.buffer_size)
    train_info = {}
    for _ in range(n_epochs):
        np.random.shuffle(indexes)
        for start in range(0, agent.buffer_size, agent.batch_size):
            end = start + agent.batch_size
            sample_idx = indexes[start:end]
            samples = agent.memory.sample(sample_idx)
            train_info = agent.learner.update(**samples)
    return train_info
