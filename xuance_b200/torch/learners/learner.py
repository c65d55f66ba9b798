"""Learner base class - mirror of xuance/torch/learners/base/drl_learner.py:12-214.

Same constructor contract (config fields read the same way), ``update`` abstract, ``save_model`` /
``load_model`` writing/reading the reference's checkpoint dict ({'policy', 'optimizer', 'rng_state',
'cuda_rng_state'}, drl_learner.py:64-93).  Distributed training is the torchrun process group; there are no
per-module DDP wrappers, the learner all-reduces its flat gradient bucket once per update."""
import os
from abc import ABC, abstractmethod
from pathlib import Path

import torch
import torch.distributed as dist

from ... import _lib
from ..utils import allreduce_sum_, CapturedStep


class Learner(ABC):
    rank_suffix = True       # info keys get "/rank_{r}" in distributed runs; the reference's MARL learners log without it

    def __init__(self, config, model, callback):
        self.value_normalizer = None
        self.config = config
        self.distributed_training = bool(getattr(config, "distributed_training", False))
        self.episode_length = getattr(config, "episode_length", None)
        self.learning_rate = getattr(config, "learning_rate", None)
        self.use_linear_lr_decay = getattr(config, "use_linear_lr_decay", False)
        self.end_factor_lr_decay = getattr(config, "end_factor_lr_decay", 1.0)
        self.gamma = getattr(config, "gamma", 0.99)
        self.use_cnn = getattr(config, "use_cnn", False)
        self.use_rnn = getattr(config, "use_rnn", False)
        self.use_actions_mask = getattr(config, "use_actions_mask", False)
        self.model = model
        self.optimizer = None
        self.scheduler = None
        self.callback = callback
        if self.distributed_training and dist.is_available() and dist.is_initialized():
            self.world_size = dist.get_world_size()
            self.rank = dist.get_rank()
        elif self.distributed_training:
            self.world_size = int(os.environ.get("WORLD_SIZE", "1"))
            self.rank = int(os.environ.get("RANK", "0"))
        else:
            self.world_size, self.rank = 1, 0
        self.use_grad_clip = config.use_grad_clip
        self.grad_clip_norm = config.grad_clip_norm
        self.device = torch.device(config.device if not isinstance(config.device, int) else "cuda:%d" % config.device)
        if self.device.type != "cuda":
            raise RuntimeError("xuance_b200 learners run on CUDA devices only (config.device=%r); there is no "
                               "CPU fallback" % (config.device,))
        _lib.use_device(self.device)
        self.model_dir = getattr(config, "model_dir", "./models")
        self.total_iters = self.estimate_total_iterations()
        self.iterations = 0
        self.use_cuda_graph = getattr(config, "use_cuda_graph", False)
        self._graphs = {}
        # device tensors a graphed update mutates besides the FusedAdam state (target networks, running statistics):
        # the warm-up runs of a CUDA-graph capture are real, so _snapshot / _restore must cover all of them
        self._graph_tensors = []

    def estimate_total_iterations(self):
        """drl_learner.py:57-62."""
        start_training = getattr(self.config, "start_training", 0)
        training_frequency = getattr(self.config, "training_frequency", 1)
        return (self.config.running_steps - start_training) // (training_frequency * self.config.parallels)

    # ---------------------------------------------------------------- the update protocol shared by every learner
    def _f32(self, x):
        return torch.as_tensor(x, device=self.device).to(torch.float32).contiguous()

    def _linear_lr(self, optimizer, total_iters=None):
        """The reference's LinearLR schedule from 1 to ``end_factor_lr_decay`` over ``total_iters`` (default: the
        estimated update count)."""
        return torch.optim.lr_scheduler.LinearLR(optimizer, start_factor=1.0, end_factor=self.end_factor_lr_decay,
                                                 total_iters=self.total_iters if total_iters is None else total_iters)

    def _optimizer_step(self, opt, outputs, grads, inputs=None):
        """Backward of ``outputs`` seeded with ``grads`` into ``opt``'s flat bucket (restricted to ``inputs`` if given),
        ONE all-reduce of gradient + logged statistics when sharded, then the K7 clip + Adam step."""
        opt.zero_grad()
        torch.autograd.backward(outputs, grads, inputs=inputs)
        if self.world_size > 1:
            allreduce_sum_(opt.bucket.grad_all)
        opt.launch(max_norm=self.grad_clip_norm if self.use_grad_clip else None)

    def _device_step(self, key, fn, *args):
        """Runs ``fn(*args)``, the device half of an update: eagerly, or with ``use_cuda_graph`` as the replay of a graph
        captured once per ``key`` (``key=None`` runs eagerly).  Returns what ``fn`` returns (a graph's static output)."""
        if not self.use_cuda_graph or key is None:
            return fn(*args)
        if key not in self._graphs:
            self._graphs[key] = CapturedStep(fn, list(args), self._snapshot, self._restore)
        return self._graphs[key](*args)

    def _optimizers(self):
        """Every FusedAdam a device update steps."""
        return list(self.optimizer.values()) if isinstance(self.optimizer, dict) else [self.optimizer]

    def _snapshot(self):
        return [o.snapshot() for o in self._optimizers()], [t.detach().clone() for t in self._graph_tensors]

    def _restore(self, st):
        for o, s in zip(self._optimizers(), st[0]):
            o.restore(s)
        with torch.no_grad():
            for t, s in zip(self._graph_tensors, st[1]):
                t.copy_(s)

    def _with_rank(self, vals):
        if self.distributed_training and self.rank_suffix:
            return {f"{k}/rank_{self.rank}": v for k, v in vals.items()}
        return vals

    def _finish_info(self, info, vals, **models):
        """Adds an update's logged values to ``info`` and runs the callback's on_update_end (``models``: the keyword the
        reference passes the network under, ``model=`` or ``policy=``)."""
        info.update(self._with_rank(vals))
        info.update(self.callback.on_update_end(self.iterations, info=info, **models) or {})
        return info

    # ---------------------------------------------------------------- checkpoints (reference format)
    def _opt_state(self):
        if isinstance(self.optimizer, dict):
            return {k: v.state_dict() for k, v in self.optimizer.items()}
        return self.optimizer.state_dict()

    def save_model(self, model_path):
        os.makedirs(os.path.dirname(os.path.abspath(model_path)), exist_ok=True)
        torch.save({'policy': self.model.state_dict(), 'optimizer': self._opt_state(),
                    'rng_state': torch.get_rng_state(),
                    'cuda_rng_state': torch.cuda.get_rng_state_all()}, model_path)

    def load_model(self, path, model=None):
        """drl_learner.py:95-157: a file, or a directory holding seed_* folders -> newest -> final_train_model.pth
        (or any .pth).  Restores policy, optimizer and RNG state."""
        target = os.path.join(path, model) if model is not None else path
        if os.path.isfile(target):
            model_path = target
        else:
            if not os.path.isdir(path):
                raise RuntimeError(f"The path '{path}' is not a valid directory or file!")
            folders = sorted(f for f in os.listdir(path) if "seed_" in f)
            if not folders:
                raise RuntimeError(f"No model files with 'seed_' found in '{path}'!")
            d = Path(os.path.join(path, folders[-1]))
            names = list(d.glob("*.pth"))
            if not names:
                raise FileNotFoundError(f"No .pth file found in {d}")
            finals = [f for f in names if "final_train_model.pth" in str(f)]
            model_path = str(finals[0] if finals else sorted(names)[-1])
        ckpt = torch.load(str(model_path), map_location=self.device, weights_only=True)
        self.model.load_state_dict(ckpt['policy'])
        opt = ckpt.get('optimizer')
        if opt is not None:
            if isinstance(self.optimizer, dict):
                for k, v in self.optimizer.items():
                    if k in opt:
                        v.load_state_dict(opt[k])
            elif self.optimizer is not None:
                self.optimizer.load_state_dict(opt)
        self._restore_rng(ckpt)
        self._safe_scheduler_step()
        print(f"Successfully load model from '{model_path}'.")
        return model_path

    @staticmethod
    def _restore_rng(ckpt):
        """drl_learner.py:146-152 / 172-178: CPU generator and every visible device's CUDA generator."""
        if ckpt.get('rng_state') is not None:
            torch.set_rng_state(ckpt['rng_state'].cpu())
        cuda_states = ckpt.get('cuda_rng_state')
        if isinstance(cuda_states, (list, tuple)) and torch.cuda.is_available():
            for i, state in enumerate(cuda_states[:torch.cuda.device_count()]):
                torch.cuda.set_rng_state(state.cpu(), device=i)

    # ---------------------------------------------------------------- snapshots (drl_learner.py:34-44, 159-189)
    # The reference keeps ONE rolling file, <model_dir>/DDP_Snapshot/snapshot.pt, written by rank 0 and loaded by every rank
    # when a distributed learner is constructed, so an interrupted torchrun job resumes with policy, optimiser and RNG state.
    @property
    def snapshot_path(self):
        return os.path.join(os.getcwd(), self.model_dir, "DDP_Snapshot")

    def save_snapshot(self):
        if self.rank != 0:
            return None
        os.makedirs(self.snapshot_path, exist_ok=True)
        path = os.path.join(self.snapshot_path, "snapshot.pt")
        torch.save({"policy": self.model.state_dict(), "optimizer": self._opt_state(), "iterations": self.iterations,
                    "rng_state": torch.get_rng_state(), "cuda_rng_state": torch.cuda.get_rng_state_all()}, path)
        return path

    def load_snapshot(self, snapshot_path=None):
        """Accepts the snapshot directory or the file; also reads the reference's older {'MODEL_STATE': ...} layout."""
        path = self.snapshot_path if snapshot_path is None else snapshot_path
        if os.path.isdir(path):
            path = os.path.join(path, "snapshot.pt")
        snap = torch.load(path, map_location=self.device, weights_only=False)
        if "MODEL_STATE" in snap:
            self.model.load_state_dict(snap["MODEL_STATE"])
            return path
        self.model.load_state_dict(snap["policy"])
        opt = snap.get("optimizer")
        if opt is not None and self.optimizer is not None:
            if isinstance(self.optimizer, dict):
                for k, v in self.optimizer.items():
                    v.load_state_dict(opt[k])
            else:
                self.optimizer.load_state_dict(opt)
        self._restore_rng(snap)
        its = int(snap.get("iterations", 0))
        if its:                                    # resume the LinearLR schedule where the interrupted run stopped
            self.iterations = its
            self._fast_forward_scheduler(its)
        return path

    def _schedulers(self):
        sch = self.scheduler
        if sch is None:
            return []
        return list(sch.values()) if isinstance(sch, dict) else (list(sch) if isinstance(sch, list) else [sch])

    def _fast_forward_scheduler(self, current_iters):
        for sch in self._schedulers():
            sch.last_epoch = int(current_iters)
            if hasattr(sch, "_get_closed_form_lr"):             # LinearLR: lr(t) in closed form (its step() is a recurrence)
                lrs = sch._get_closed_form_lr()
                for group, lr in zip(sch.optimizer.param_groups, lrs):
                    group["lr"] = lr
                sch._last_lr = list(lrs)

    def _safe_scheduler_step(self):
        """drl_learner.py:191-210: a run restarted with ``config.rt_epoch`` (evaluation epochs already done) moves the
        learning-rate schedule to the matching iteration."""
        if not hasattr(self.config, "rt_epoch") or not self._schedulers():
            return
        try:
            train_steps = self.config.running_steps // self.config.parallels
            eval_interval = self.config.eval_interval // self.config.parallels
            num_epoch = int(train_steps / eval_interval)
            self._fast_forward_scheduler(int(self.total_iters * self.config.rt_epoch / num_epoch))
        except Exception as e:                     # the reference swallows this too (prints and carries on)
            print(f"scheduler fast-forward skipped: {e}")

    @abstractmethod
    def update(self, *args):
        raise NotImplementedError
