"""CPU: the drop-in restatement of the reference's agent loop.  The reference's own ``OnPolicyAgent.train_epochs``
(on_policy.py:182-205) and its restatement in oracle/agents.py drive recording fakes with the same NumPy seed and must
produce identical call sequences (the reference's sequence is recorded in tests/golden/reference_live.pkl.gz by
tests/golden/make_reference_live.py).  tests/test_gpu_dropin.py then runs that restatement over the real xuance_b200
buffer + learner on the GPU."""
import gzip
import os
import pickle
from types import SimpleNamespace

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class _Recorder:
    def __init__(self):
        self.calls = []

    def sample(self, idx):
        self.calls.append(("sample", np.array(idx, copy=True)))
        return {"obs": idx[:1], "actions": idx[:1], "returns": idx[:1], "values": idx[:1], "advantages": idx[:1],
                "aux_batch": {}, "batch_size": len(idx)}

    def update(self, **samples):
        self.calls.append(("update", tuple(sorted(samples))))
        return {"n": len(self.calls)}


@pytest.mark.parametrize("buffer_size,batch_size,n_epochs", [(64, 16, 4), (60, 16, 3)])
def test_train_epochs_restatement_equals_the_live_reference(buffer_size, batch_size, n_epochs):
    from oracle.agents import reference_train_epochs
    with gzip.open(os.path.join(ROOT, "tests", "golden", "reference_live.pkl.gz"), "rb") as fh:
        want = pickle.load(fh)["train_epochs"][(buffer_size, batch_size, n_epochs)]
    rec = _Recorder()
    agent = SimpleNamespace(buffer_size=buffer_size, batch_size=batch_size, memory=rec, learner=rec)
    np.random.seed(11)
    info = reference_train_epochs(agent, n_epochs)
    a, ia, b, ib = want["calls"], want["info"], rec.calls, info
    assert ia == ib and len(a) == len(b) and len(a) == 2 * n_epochs * -(-buffer_size // batch_size)
    for (ka, va), (kb, vb) in zip(a, b):
        assert ka == kb and (np.array_equal(va, vb) if ka == "sample" else va == vb)
