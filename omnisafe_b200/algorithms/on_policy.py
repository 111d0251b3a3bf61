"""On-policy algorithms on the fused sm_90a path: PolicyGradient / PPO / PPOLag / NaturalPG / RCPO /
TRPO / TRPOLag / CPO / PCPO / FOCOPS / CPPOPID / TRPOPID / OnCRPO / PDO / IPO / P3O.

Each class mirrors the override structure of the reference
(omnisafe/algorithms/on_policy/base/{policy_gradient,ppo,natural_pg,trpo}.py,
naive_lagrange/{ppo_lag,trpo_lag}.py, second_order/cpo.py, first_order/focops.py): the same
`_init_env/_init_model/_init/_init_log/learn/_update/_update_actor` hooks and logger keys, with the
method bodies handing the work to the C-ABI kernels (rollout, dual GAE, fused update, CG/FVP).
"""
from __future__ import annotations

import math
import time

import torch

from omnisafe_b200.adapter.onpolicy_adapter import OnPolicyAdapter
from omnisafe_b200.adapter.early_terminated_adapter import EarlyTerminatedAdapter, ExternalEarlyTerminatedAdapter
from omnisafe_b200.adapter.external_adapter import ExternalEnvAdapter
from omnisafe_b200.adapter.saute_adapter import SauteAdapter
from omnisafe_b200.adapter.simmer_adapter import SimmerAdapter
from omnisafe_b200.algorithms import registry
from omnisafe_b200.algorithms.base_algo import BaseAlgo
from omnisafe_b200.algorithms.engine import (LOSS_COST, LOSS_FOCOPS, LOSS_P3O, LOSS_PPO_CLIP, LOSS_RATIO,
                                             NET_ACTOR, UpdateEngine)
from omnisafe_b200.common.buffer import VectorOnPolicyBuffer
from omnisafe_b200.common.lagrange import Lagrange
from omnisafe_b200.common.logger import Logger
from omnisafe_b200.common.pid_lagrange import PIDLagrangian
from omnisafe_b200.envs.synthetic import support_envs as synthetic_envs
from omnisafe_b200.models.actor_critic import ConstraintActorCritic
from omnisafe_b200.utils import distributed, train_state


def _plain_adapter(env_id: str):
    """The synthetic env runs inside the fused rollout kernel; a registered CMDP is stepped in PyTorch around the
    act / observe kernels."""
    return OnPolicyAdapter if env_id in synthetic_envs() else ExternalEnvAdapter


def _require_synthetic(env_id: str, what: str) -> None:
    if env_id not in synthetic_envs():
        raise NotImplementedError(f'{what} runs on the synthetic env only; {env_id} is a registered external env')


@registry.register
class PolicyGradient(BaseAlgo):
    """base/policy_gradient.py:L39-588."""

    _loss_kind = LOSS_RATIO

    # ---- construction ------------------------------------------------------------------------
    def _init_env(self) -> None:
        t, a = self._cfgs.train_cfgs, self._cfgs.algo_cfgs
        rank = distributed.get_rank()
        self._env = _plain_adapter(self._env_id)(self._env_id, t.vector_env_nums, self._seed, self._cfgs,
                                                 device=self._device, env_id_offset=rank * t.vector_env_nums)
        self._steps_per_epoch = distributed.local_steps(a.steps_per_epoch, t.vector_env_nums)

    def _init_model(self) -> None:
        gen = torch.Generator().manual_seed(int(self._cfgs.seed))   # identical on every rank == sync_params
        self._actor_critic = ConstraintActorCritic(self._env.obs_dim, self._env.act_dim, self._cfgs.model_cfgs,
                                                   epochs=self._cfgs.train_cfgs.epochs, device=self._device,
                                                   generator=gen)

    def _init(self) -> None:
        a = self._cfgs.algo_cfgs
        self._buf = VectorOnPolicyBuffer(
            self._env.obs_dim, self._env.act_dim, self._steps_per_epoch, a.gamma, a.lam, a.lam_c,
            a.adv_estimation_method, a.penalty_coef, a.standardized_rew_adv, a.standardized_cost_adv,
            num_envs=self._cfgs.train_cfgs.vector_env_nums, device=self._device, keep_discounted_ret=False)
        self._engine = UpdateEngine(self._actor_critic, self._buf)
        prec = str(getattr(self._cfgs.train_cfgs, 'matmul_precision', 'bf16x3'))   # upstream YAMLs have no such key: parity-grade tensor-core tiles
        assert prec in ('fp32', 'tf32', 'bf16x3'), "train_cfgs.matmul_precision must be 'fp32', 'tf32' or 'bf16x3'"
        self._engine.precision = {'fp32': 0, 'tf32': 1, 'bf16x3': 2}[prec]
        self._actor_critic.precision = self._engine.precision   # step / predict / critics use the training arithmetic
        self._stats8 = torch.zeros(8, dtype=torch.float64, device=self._device)
        self._epochs_done = 0       # epochs trained so far (a resumed run starts at the saved count)
        self._first_epoch = 0       # where learn() starts

    def _init_log(self) -> None:
        lc = self._cfgs.logger_cfgs
        self._logger = Logger(lc.log_dir, self._cfgs.exp_name, seed=self._cfgs.seed, config=self._cfgs,
                              verbose=bool(getattr(lc, 'verbose', False)), run_dir=self._run_dir)
        what = {'pi': self._actor_critic.actor_state_dict}
        what.update(self._env.save())
        self._logger.setup_torch_saver(what)
        for key in ('Metrics/EpRet', 'Metrics/EpCost', 'Metrics/EpLen', 'Train/Epoch', 'Train/Entropy',
                    'Train/KL', 'Train/StopIter', 'Train/PolicyRatio', 'Train/LR', 'Train/PolicyStd',
                    'TotalEnvSteps', 'Loss/Loss_pi', 'Loss/Loss_reward_critic', 'Loss/Loss_cost_critic',
                    'Time/Total', 'Time/Rollout', 'Time/Update', 'Time/Epoch', 'Time/FPS'):
            self._logger.register_key(key)

    # ---- training loop (policy_gradient.py:L238-306) -------------------------------------------
    def learn(self, save_state_freq: int = 0) -> tuple[float, float, float]:
        """Train epochs `_first_epoch` (0, or k after `load_train_state`) .. epochs-1.  `save_state_freq` > 0: write the
        training state after every `save_state_freq`-th epoch and after the last one."""
        self._start_time = time.time()
        t = self._cfgs.train_cfgs
        for epoch in range(self._first_epoch, t.epochs):
            self.train_epoch(log=True, epoch=epoch)
            if (epoch + 1) % self._cfgs.logger_cfgs.save_model_freq == 0 or (epoch + 1) == t.epochs:
                self._logger.torch_save()
            if save_state_freq > 0 and ((epoch + 1) % save_state_freq == 0 or (epoch + 1) == t.epochs):
                self.save_train_state()
        ep = self._window_means()
        self._logger.close()
        self._env.close()
        return ep

    def train_epoch(self, eps=None, log: bool = False, epoch: int | None = None):
        """One epoch: rollout -> dual GAE -> statistics exchange -> update.  Asynchronous unless
        `log` (the logger reads the epoch's metrics back, one synchronisation per epoch).  `eps`
        optionally supplies the [T, N, A] standard-normal stream (parity mode)."""
        epoch_time = time.time()
        self._env.rollout(self._steps_per_epoch, self._actor_critic, self._buf, self._logger, eps=eps)
        self._buf.finish_paths()
        self._reduce_epoch_statistics()
        roll = time.time()
        self._update()
        self._actor_critic.actor_scheduler_step()
        self._epochs_done += 1
        if not log:
            self._epochs_unchecked = getattr(self, '_epochs_unchecked', 0) + 1
            if distributed.world_size() > 1 and self._epochs_unchecked >= 16:     # the NVLink exchange reports time-outs through a flag
                self._epochs_unchecked = 0
                distributed.p2p_check()
            return None
        if epoch is None:
            epoch = self._logger.current_epoch
        return self._log_epoch(epoch, getattr(self, '_start_time', epoch_time), epoch_time, roll)

    def _reduce_epoch_statistics(self) -> None:
        """The once-per-epoch exchange: {adv sums, episode-window sums} in one fp64 all-reduce
        (vector_onpolicy_buffer.py:L131-132 + logger.py:L365-373), then the advantage moments."""
        if distributed.world_size() > 1:
            self._stats8[:4] = self._buf.adv_sums
            self._stats8[4:] = self._env.window_sums
            distributed.all_reduce_(self._stats8)
            self._buf.adv_sums.copy_(self._stats8[:4])
            self._env.window_sums.copy_(self._stats8[4:])
        self._buf.finalize_statistics()

    def _window_means(self) -> tuple[float, float, float]:
        ws = self._env.window_sums.tolist()
        n = ws[3] if ws[3] > 0 else float('nan')
        return ws[0] / n, ws[1] / n, ws[2] / n

    def _log_epoch(self, epoch, start, epoch_time, roll) -> None:
        torch.cuda.synchronize()
        distributed.p2p_check()
        now = time.time()
        ep_ret, ep_cost, ep_len = self._window_means()
        ts = self._engine.train_stats.view(3, 8).tolist()
        kl = self._engine.kl_state.tolist()
        n_mb = [max(r[3], 1.0) for r in ts]
        std = float(torch.exp(self._actor_critic.theta[: self._env.act_dim]).mean())
        logstd = float(self._actor_critic.theta[: self._env.act_dim].mean())
        gsteps = self._cfgs.algo_cfgs.steps_per_epoch
        self._logger.store({
            'Metrics/EpRet': ep_ret, 'Metrics/EpCost': ep_cost, 'Metrics/EpLen': ep_len,
            'Train/Epoch': epoch, 'Train/Entropy': 0.5 + 0.5 * math.log(2 * math.pi) + logstd,
            'Train/KL': kl[0], 'Train/StopIter': kl[1], 'Train/PolicyRatio': ts[0][1] / n_mb[0],
            'Train/LR': self._actor_critic.actor_lr, 'Train/PolicyStd': std,
            'TotalEnvSteps': (epoch + 1) * gsteps, 'Loss/Loss_pi': ts[0][0] / n_mb[0],
            'Loss/Loss_reward_critic': ts[1][0] / n_mb[1], 'Loss/Loss_cost_critic': ts[2][0] / n_mb[2],
            'Time/Total': now - start, 'Time/Rollout': roll - epoch_time, 'Time/Update': now - roll,
            'Time/Epoch': now - epoch_time, 'Time/FPS': gsteps / (now - epoch_time),
        })
        self._log_extra()
        self._logger.dump_tabular()
        A = self._env.act_dim
        return {'d2h_bytes': 4 * 8 + 24 * 4 + 4 * 4 + 2 * A * 4 + 8, 'fps': gsteps / (now - epoch_time)}

    def _log_extra(self) -> None:
        pass

    # ---- training state: save at an epoch boundary, resume bit for bit ---------------------------------------------------
    def _state_meta(self) -> dict:
        return {**train_state.config_meta(self._cfgs, distributed.world_size()), 'obs_dim': self._env.obs_dim,
                'act_dim': self._env.act_dim}

    def _train_state(self) -> dict:
        """This rank's state, composed from the owners' train_state() (subclasses add their own entries).  The global
        RNGs are part of it: the policy step's sampling and user envs draw from them."""
        return {'epochs_done': self._epochs_done, 'model': self._actor_critic.train_state(),
                'engine': self._engine.train_state(), 'env': self._env.train_state(),
                'logger': self._logger.train_state(),
                'rng': {'cpu': torch.get_rng_state(), 'cuda': torch.cuda.get_rng_state(self._device)}}

    def _load_train_state(self, state: dict) -> None:
        self._actor_critic.load_train_state(state['model'])
        self._engine.load_train_state(state['engine'])
        self._env.load_train_state(state['env'])
        self._logger.load_train_state(state['logger'])
        torch.set_rng_state(state['rng']['cpu'])
        torch.cuda.set_rng_state(state['rng']['cuda'], self._device)
        self._epochs_done = self._first_epoch = int(state['epochs_done'])

    def save_train_state(self) -> str:
        """Write every rank's training state to <log_dir>/train_state/epoch-{k}/ (k = epochs trained) and return the
        directory.  Call it between epochs; every rank must call it."""
        k = self._epochs_done
        rank = distributed.get_rank()
        sdir = distributed.broadcast_object(train_state.state_dir(self._logger.log_dir, k))
        if rank == 0:
            train_state.begin(sdir)
        distributed.barrier()
        train_state.write_rank(sdir, rank, k, self._train_state())
        distributed.barrier()
        if rank == 0:
            train_state.write_meta(sdir, {**self._state_meta(), 'epoch': k})
        distributed.barrier()
        return sdir

    def load_train_state(self, sdir: str) -> None:
        """Load this rank's state from a directory `save_train_state` wrote, into the tensors this object allocated."""
        meta = train_state.read_meta(sdir)
        train_state.check_meta(meta, self._state_meta(), sdir)
        self._load_train_state(train_state.load_rank(sdir, distributed.get_rank(), int(meta['epoch'])))

    # ---- update (policy_gradient.py:L308-405) -----------------------------------------------------
    def _lagrange_ptr(self):
        return None

    def _update(self, net_mask: int = 7, perm=None) -> None:
        a = self._cfgs.algo_cfgs
        if not a.use_cost:
            net_mask &= ~4
        self._engine.ppo_epoch(
            loss_kind=self._loss_kind, lagrange=self._lagrange_ptr(), net_mask=net_mask,
            batch_size=a.batch_size, update_iters=a.update_iters, clip=getattr(a, 'clip', 0.2),
            entropy_coef=a.entropy_coef, focops_lam=getattr(a, 'focops_lam', 1.0),
            focops_eta=getattr(a, 'focops_eta', 0.0),
            critic_norm_coef=a.critic_norm_coef if a.use_critic_norm else 0.0,
            max_grad_norm=a.max_grad_norm if a.use_max_grad_norm else 0.0,
            lr_actor=self._actor_critic.actor_lr, lr_critic=self._actor_critic.critic_lr,
            target_kl=a.target_kl, kl_early_stop=a.kl_early_stop, perm=perm)


@registry.register
class PPO(PolicyGradient):
    """base/ppo.py:L28-87 (clipped surrogate)."""

    _loss_kind = LOSS_PPO_CLIP


class _LagrangeMixin:
    """The `_init / _init_log / _update` additions shared by PPOLag / TRPOLag / FOCOPS
    (naive_lagrange/ppo_lag.py:L31-80)."""

    def _init(self) -> None:
        super()._init()
        self._lagrange = Lagrange(**self._cfgs.lagrange_cfgs.todict(), device=self._device)

    def _init_log(self) -> None:
        super()._init_log()
        self._logger.register_key('Metrics/LagrangeMultiplier')

    def _lagrange_ptr(self):
        return self._lagrange.state

    def _train_state(self) -> dict:
        return {**super()._train_state(), 'lagrange': self._lagrange.train_state()}

    def _load_train_state(self, state: dict) -> None:
        super()._load_train_state(state)
        self._lagrange.load_train_state(state['lagrange'])

    def _update(self, *args, **kwargs) -> None:
        # Jc = windowed mean EpCost (already all-reduced); first update lambda, then the networks
        self._lagrange.update_lagrange_multiplier(self._env.window_sums)
        super()._update(*args, **kwargs)

    def _log_extra(self) -> None:
        super()._log_extra()
        assert int(self._lagrange.nan_flag) == 0, 'cost for updating lagrange multiplier is nan'
        self._logger.store({'Metrics/LagrangeMultiplier': float(self._lagrange.lagrangian_multiplier)})


@registry.register
class PPOLag(_LagrangeMixin, PPO):
    """naive_lagrange/ppo_lag.py:L26-102."""


@registry.register
class PDO(_LagrangeMixin, PolicyGradient):
    """naive_lagrange/pdo.py:L25-100: PolicyGradient on the Lagrangian surrogate (its YAML defaults switch
    the reward / cost normalisers on)."""


@registry.register
class IPO(PPO):
    """penalty_function/ipo.py:L24-74: PPO on (adv_r - penalty adv_c) / (1 + penalty) with the interior-point
    penalty kappa / (cost_limit - Jc + 1e-8), replaced by penalty_max when negative or too large."""

    def _init(self) -> None:
        super()._init()
        self._penalty_state = torch.zeros(4, dtype=torch.float32, device=self._device)
        self._penalty = 0.0

    def _init_log(self) -> None:
        super()._init_log()
        self._logger.register_key('Misc/Penalty')

    def _lagrange_ptr(self):
        return self._penalty_state

    def _train_state(self) -> dict:
        return {**super()._train_state(), 'penalty_state': self._penalty_state.cpu().clone(), 'penalty': self._penalty}

    def _load_train_state(self, state: dict) -> None:
        super()._load_train_state(state)
        train_state.restore(self._penalty_state, state['penalty_state'], 'IPO penalty state')
        self._penalty = float(state['penalty'])

    def _update(self, *args, **kwargs) -> None:
        a = self._cfgs.algo_cfgs
        jc = self._window_means()[1]            # the reference reads the logger here too (ipo.py:L68)
        penalty = a.kappa / (a.cost_limit - jc + 1e-8)
        if penalty < 0 or penalty > a.penalty_max:
            penalty = a.penalty_max
        self._penalty = float(penalty)
        self._penalty_state[0] = self._penalty
        super()._update(*args, **kwargs)

    def _log_extra(self) -> None:
        super()._log_extra()
        self._logger.store({'Misc/Penalty': self._penalty})


@registry.register
class P3O(PPO):
    """penalty_function/p3o.py:L29-125: the PPO clipped surrogate on adv_r plus the exact penalty
    kappa * relu(mean(ratio adv_c) + Jc - cost_limit) in the actor loss."""

    _loss_kind = LOSS_P3O

    def _init_log(self) -> None:
        super()._init_log()
        self._logger.register_key('Loss/Loss_pi_cost', delta=True)

    def _update(self, net_mask: int = 7, perm=None) -> None:
        a = self._cfgs.algo_cfgs
        jc = self._window_means()[1] - a.cost_limit        # the reference reads the logger per minibatch (p3o.py:L88)
        self._engine.ppo_epoch(
            loss_kind=LOSS_P3O, lagrange=None, net_mask=net_mask if a.use_cost else net_mask & ~4,
            batch_size=a.batch_size, update_iters=a.update_iters, clip=a.clip, entropy_coef=a.entropy_coef,
            focops_lam=a.kappa, focops_eta=jc,
            critic_norm_coef=a.critic_norm_coef if a.use_critic_norm else 0.0,
            max_grad_norm=a.max_grad_norm if a.use_max_grad_norm else 0.0,
            lr_actor=self._actor_critic.actor_lr, lr_critic=self._actor_critic.critic_lr,
            target_kl=a.target_kl, kl_early_stop=a.kl_early_stop, perm=perm)

    def _log_extra(self) -> None:
        super()._log_extra()
        ts = self._engine.train_stats[:8].tolist()      # actor slots: loss, ratio, penalty term, minibatch steps
        self._logger.store({'Loss/Loss_pi_cost': ts[2] / max(ts[3], 1.0)})


@registry.register
class FOCOPS(_LagrangeMixin, PolicyGradient):
    """first_order/focops.py:L31-230."""

    _loss_kind = LOSS_FOCOPS


@registry.register
class NaturalPG(PolicyGradient):
    """base/natural_pg.py:L30-230: one full-batch natural-gradient actor step, then critic passes."""

    _kind = LOSS_RATIO

    def _init_log(self) -> None:
        super()._init_log()
        for key in ('Misc/Alpha', 'Misc/FinalStepNorm', 'Misc/gradient_norm', 'Misc/xHx', 'Misc/H_inv_g'):
            self._logger.register_key(key)
        self._misc: dict[str, float] = {}

    def _log_extra(self) -> None:
        super()._log_extra()
        self._logger.store(self._misc)

    def _adv_lagrange(self):
        return self._lagrange_ptr()

    def _surrogate_kind(self) -> int:
        """Which actor loss `_loss_pi(obs, act, logp, adv)` stands for this epoch: LOSS_RATIO with
        adv = _compute_adv_surrogate(adv_r, adv_c), or LOSS_COST when the surrogate is -adv_c (OnCRPO)."""
        return LOSS_RATIO

    def _natural_direction(self):
        """theta_old, g = -grad(loss), x = H^-1 g, xHx, alpha (natural_pg.py:L146-166)."""
        a, e, ac = self._cfgs.algo_cfgs, self._engine, self._actor_critic
        Pa = e.Pa
        e.snapshot_old_policy()
        theta_old = ac.theta[:Pa].clone()
        grads = torch.empty(Pa, dtype=torch.float32, device=self._device)
        self._kind = self._surrogate_kind()
        loss_before = e.actor_loss_grad(self._kind, self._adv_lagrange(), grads, sign=-1.0)
        x = e.conjugate_gradients(grads, a.cg_iters, a.cg_damping, a.fvp_sample_freq)
        assert torch.isfinite(x).all(), 'x is not finite'
        e.fvp(x, e.cg_z, a.cg_damping, a.fvp_sample_freq)
        xHx = e.dot(x, e.cg_z)
        assert xHx >= 0, 'xHx is negative'
        alpha = math.sqrt(2 * a.target_kl / (xHx + 1e-8))
        return theta_old, grads, x, xHx, alpha, float(loss_before)

    def _update_actor(self) -> None:
        theta_old, grads, x, xHx, alpha, _ = self._natural_direction()
        step = alpha * x
        self._actor_critic.theta[: self._engine.Pa] = theta_old + step
        self._misc = {'Misc/Alpha': alpha, 'Misc/FinalStepNorm': float(step.norm()), 'Misc/xHx': xHx,
                      'Misc/gradient_norm': float(grads.norm()), 'Misc/H_inv_g': float(x.norm())}

    def _update(self, perm=None) -> None:
        self._update_actor()
        final_kl = self._engine.kl_state[0].clone()
        super()._update(net_mask=6, perm=perm)   # critics only, update_iters passes (natural_pg.py:L209-223)
        # what the reference logs after the actor step (natural_pg.py:L168-186, trpo.py:L196-222): loss / ratio / KL of
        # the accepted policy on the full batch, StopIter = update_iters
        ev = self._engine.evaluate(self._actor_critic.theta, self._adv_lagrange())
        ts = self._engine.train_stats.view(3, 8)
        ts[0, 0] = ev['loss_c'] if self._kind == LOSS_COST else ev['loss']
        ts[0, 1] = ev['ratio']
        ts[0, 3] = 1.0
        self._engine.kl_state[0] = final_kl if float(final_kl) != 0.0 else ev['kl']
        self._engine.kl_state[1] = float(self._cfgs.algo_cfgs.update_iters)


@registry.register
class RCPO(_LagrangeMixin, NaturalPG):
    """naive_lagrange/rcpo.py:L25-103 (natural gradient step on the Lagrangian surrogate)."""


@registry.register
class TRPO(NaturalPG):
    """base/trpo.py:L32-222: natural direction + backtracking line search."""

    def _init_log(self) -> None:
        super()._init_log()
        self._logger.register_key('Misc/AcceptanceStep')

    def _search_step_size(self, step_direction, grads, theta_old, loss_before, total_steps=15, decay=0.8):
        a, e = self._cfgs.algo_cfgs, self._engine
        step_frac, final_kl = 1.0, 0.0
        trial = self._actor_critic.theta.clone()
        acceptance_step = 0
        for step in range(total_steps):
            trial[: e.Pa] = theta_old + step_frac * step_direction
            ev = e.evaluate(trial, self._adv_lagrange())
            loss = ev['loss_c'] if self._kind == LOSS_COST else ev['loss']
            loss_improve = loss_before - loss
            if not math.isfinite(loss):
                self._logger.log('WARNING: loss_pi not finite')
            elif loss_improve < 0:
                self._logger.log('INFO: did not improve improve <0')
            elif ev['kl'] > a.target_kl:
                self._logger.log('INFO: violated KL constraint.')
            else:
                acceptance_step, final_kl = step + 1, ev['kl']
                break
            step_frac *= decay
        else:
            self._logger.log('INFO: no suitable step found...')
            step_direction = torch.zeros_like(step_direction)
        self._engine.kl_state[0] = final_kl
        return step_frac * step_direction, acceptance_step

    def _update_actor(self) -> None:
        theta_old, grads, x, xHx, alpha, loss_before = self._natural_direction()
        step, accept = self._search_step_size(alpha * x, grads, theta_old, loss_before)
        self._actor_critic.theta[: self._engine.Pa] = theta_old + step
        self._misc = {'Misc/Alpha': alpha, 'Misc/FinalStepNorm': float(step.norm()), 'Misc/xHx': xHx,
                      'Misc/gradient_norm': float(grads.norm()), 'Misc/H_inv_g': float(x.norm()),
                      'Misc/AcceptanceStep': accept}


@registry.register
class TRPOLag(_LagrangeMixin, TRPO):
    """naive_lagrange/trpo_lag.py:L25-103."""


@registry.register
class CPO(TRPO):
    """second_order/cpo.py:L33-462."""

    def _init_log(self) -> None:
        super()._init_log()
        for key in ('Misc/cost_gradient_norm', 'Misc/Lambda_star', 'Misc/Nu_star', 'Misc/OptimCase',
                    'Misc/A', 'Misc/B', 'Misc/q', 'Misc/r', 'Misc/s'):
            self._logger.register_key(key)

    def _adv_lagrange(self):
        return None   # CPO's reward surrogate uses adv_r alone

    def _determine_case(self, b_dot_b, ep_costs, q, r, s):
        kl = self._cfgs.algo_cfgs.target_kl
        if b_dot_b <= 1e-6 and ep_costs < 0:
            return 4, 0.0, 0.0
        assert math.isfinite(r), 'r is not finite'
        assert math.isfinite(s), 's is not finite'
        A = q - r ** 2 / (s + 1e-8)
        B = 2 * kl - ep_costs ** 2 / (s + 1e-8)
        if ep_costs < 0 and B < 0:
            return 3, A, B
        if ep_costs < 0 <= B:
            return 2, A, B
        if ep_costs >= 0 and B >= 0:
            self._logger.log('Alert! Attempting feasible recovery!')
            return 1, A, B
        self._logger.log('Alert! Attempting infeasible recovery!')
        return 0, A, B

    def _step_direction(self, optim_case, xHx, x, A, B, q, p, r, s, ep_costs):
        """second_order/cpo.py:L271-337.  The reference evaluates these scalars as fp32 tensors, i.e. with IEEE
        semantics: sqrt of a negative number (A = q - r^2/s can come out slightly negative after an inexact CG solve)
        and x / 0 give NaN / inf instead of raising, a NaN comparison is False, so the search falls back to
        lambda_b_star or a zero step.  `_sqrt` / `_div` reproduce that instead of Python's exceptions."""
        kl = self._cfgs.algo_cfgs.target_kl
        nan, inf = float('nan'), math.inf
        _sqrt = lambda v: math.sqrt(v) if v >= 0 else nan   # noqa: E731  (NaN input: comparison False -> NaN)

        def _div(a, b):
            if b != 0:
                return a / b
            return nan if (a == 0 or a != a) else math.copysign(inf, a) * math.copysign(1.0, b)

        def clampf(v, lo, hi):      # torch.clamp: NaN stays NaN
            return v if v != v else min(max(v, lo), hi)

        if optim_case in (3, 4):
            alpha = _sqrt(_div(2 * kl, xHx + 1e-8))
            return alpha * x, _div(1.0, alpha + 1e-8), 0.0
        if optim_case in (1, 2):
            lambda_a = _sqrt(_div(A, B))
            lambda_b = _sqrt(_div(q, 2 * kl))
            bound = _div(r, ep_costs + 1e-8)
            if ep_costs < 0:
                lambda_a_star, lambda_b_star = clampf(lambda_a, 0.0, bound), clampf(lambda_b, bound, inf)
            else:
                lambda_a_star, lambda_b_star = clampf(lambda_a, bound, inf), clampf(lambda_b, 0.0, bound)
            f_a = lambda lam: -0.5 * (_div(A, lam + 1e-8) + B * lam) - _div(r * ep_costs, s + 1e-8)   # noqa: E731
            f_b = lambda lam: -0.5 * (_div(q, lam + 1e-8) + 2 * kl * lam)   # noqa: E731
            lambda_star = lambda_a_star if f_a(lambda_a_star) >= f_b(lambda_b_star) else lambda_b_star
            nu_star = _div(max(lambda_star * ep_costs - r, 0.0), s + 1e-8)
            return _div(1.0, lambda_star + 1e-8) * (x - nu_star * p), lambda_star, nu_star
        nu_star = _sqrt(_div(2 * kl, s + 1e-8))
        return -nu_star * p, 0.0, nu_star

    def _cpo_search_step(self, step_direction, theta_old, loss_reward_before, loss_cost_before,
                         total_steps=15, decay=0.8, violation_c=0.0, optim_case=0):
        a, e = self._cfgs.algo_cfgs, self._engine
        step_frac, kl = 1.0, 0.0
        trial = self._actor_critic.theta.clone()
        acceptance_step = 0
        for step in range(total_steps):
            trial[: e.Pa] = theta_old + step_frac * step_direction
            acceptance_step = step + 1
            ev = e.evaluate(trial, None)
            kl = ev['kl']
            loss_reward_improve = loss_reward_before - ev['loss_r']
            loss_cost_diff = ev['loss_c'] - loss_cost_before
            if not math.isfinite(kl):
                self._logger.log('WARNING: KL not finite')
                continue
            if optim_case > 1 and loss_reward_improve < 0:
                self._logger.log('INFO: did not improve improve <0')
            elif loss_cost_diff > max(-violation_c, 0):
                self._logger.log(f'INFO: no improve {loss_cost_diff} > {max(-violation_c, 0)}')
            elif kl > a.target_kl:
                self._logger.log(f'INFO: violated KL constraint {kl} at step {step + 1}.')
            else:
                break
            step_frac *= decay
        else:
            self._logger.log('INFO: no suitable step found...')
            step_direction = torch.zeros_like(step_direction)
            acceptance_step = 0
        self._engine.kl_state[0] = kl
        return step_frac * step_direction, acceptance_step

    def _update_actor(self) -> None:
        a, e = self._cfgs.algo_cfgs, self._engine
        theta_old, grads, x, xHx, alpha, loss_reward_before = self._natural_direction()
        b_grads = torch.empty(e.Pa, dtype=torch.float32, device=self._device)
        loss_cost_before = float(e.actor_loss_grad(LOSS_COST, None, b_grads, sign=1.0))
        ep_costs = self._window_means()[1] - a.cost_limit
        p = e.conjugate_gradients(b_grads, a.cg_iters, a.cg_damping, a.fvp_sample_freq)
        q, r, s = xHx, e.dot(grads, p), e.dot(b_grads, p)
        optim_case, A, B = self._determine_case(e.dot(b_grads, b_grads), ep_costs, q, r, s)
        step_direction, lambda_star, nu_star = self._step_direction(optim_case, xHx, x, A, B, q, p, r, s, ep_costs)
        step, accept = self._cpo_search_step(step_direction, theta_old, loss_reward_before, loss_cost_before,
                                             total_steps=20, violation_c=ep_costs, optim_case=optim_case)
        self._actor_critic.theta[: e.Pa] = theta_old + step
        self._misc = {
            'Misc/AcceptanceStep': accept, 'Misc/Alpha': alpha, 'Misc/FinalStepNorm': float(step.norm()),
            'Misc/xHx': xHx, 'Misc/H_inv_g': float(x.norm()), 'Misc/gradient_norm': float(grads.norm()),
            'Misc/cost_gradient_norm': float(b_grads.norm()), 'Misc/Lambda_star': lambda_star,
            'Misc/Nu_star': nu_star, 'Misc/OptimCase': int(optim_case), 'Misc/A': A, 'Misc/B': B,
            'Misc/q': q, 'Misc/r': r, 'Misc/s': s}


@registry.register
class PCPO(CPO):
    """second_order/pcpo.py:L31-152: CPO's machinery with the projection step
    sqrt(2 delta / q) H x - max(0, (sqrt(2 delta / q) r + c) / s) p, searched over up to 200 halvings."""

    def _update_actor(self) -> None:
        a, e = self._cfgs.algo_cfgs, self._engine
        theta_old, grads, x, xHx, alpha, loss_reward_before = self._natural_direction()
        h_inv_g = e.cg_z.clone()                     # the reference's `H_inv_g = self._fvp(x)` (pcpo.py:L80)
        b_grads = torch.empty(e.Pa, dtype=torch.float32, device=self._device)
        loss_cost_before = float(e.actor_loss_grad(LOSS_COST, None, b_grads, sign=1.0))
        ep_costs = self._window_means()[1] - a.cost_limit
        p = e.conjugate_gradients(b_grads, a.cg_iters, a.cg_damping, a.fvp_sample_freq)
        q, r, s = xHx, e.dot(grads, p), e.dot(b_grads, p)
        f32 = lambda v: torch.tensor(v, dtype=torch.float32)   # noqa: E731  (0-dim fp32 arithmetic as in the reference)
        kl2 = 2 * a.target_kl
        coef_h = float(torch.sqrt(kl2 / (f32(q) + 1e-8)))
        coef_p = float(torch.clamp_min((torch.sqrt(kl2 / f32(q)) * f32(r) + ep_costs) / f32(s), 0.0))
        step_direction = coef_h * h_inv_g - coef_p * p
        step, accept = self._cpo_search_step(step_direction, theta_old, loss_reward_before, loss_cost_before,
                                             total_steps=200, violation_c=ep_costs)
        self._actor_critic.theta[: e.Pa] = theta_old + step
        self._misc = {
            'Misc/AcceptanceStep': accept, 'Misc/Alpha': alpha, 'Misc/FinalStepNorm': float(step.norm()),
            'Misc/xHx': xHx, 'Misc/H_inv_g': float(x.norm()), 'Misc/gradient_norm': float(grads.norm()),
            'Misc/cost_gradient_norm': float(b_grads.norm()), 'Misc/Lambda_star': 1.0, 'Misc/Nu_star': 1.0,
            'Misc/OptimCase': 1, 'Misc/A': 1.0, 'Misc/B': 1.0, 'Misc/q': q, 'Misc/r': r, 'Misc/s': s}


class _PIDLagrangeMixin(_LagrangeMixin):
    """`_init` of CPPOPID / TRPOPID (pid_lagrange/cppo_pid.py:L36-43): the multiplier is driven by the PID
    controller; `_update` (Jc -> pid_update -> super()._update()) and the surrogate
    (adv_r - lambda adv_c) / (1 + lambda) are those of the Lagrange mixin."""

    def _init(self) -> None:
        super(_LagrangeMixin, self)._init()     # skip the Adam-multiplier constructor of the Lagrange mixin
        self._lagrange = PIDLagrangian(**self._cfgs.lagrange_cfgs.todict(), device=self._device)


@registry.register
class CPPOPID(_PIDLagrangeMixin, PPO):
    """pid_lagrange/cppo_pid.py:L27-103."""


@registry.register
class TRPOPID(_PIDLagrangeMixin, TRPO):
    """pid_lagrange/trpo_pid.py:L26-103."""


@registry.register
class OnCRPO(TRPO):
    """primal/crpo.py:L25-80: TRPO on adv_r while Jc <= cost_limit + distance, otherwise on -adv_c."""

    def _init(self) -> None:
        super()._init()
        self._rew_update, self._cost_update = 0, 0

    def _init_log(self) -> None:
        super()._init_log()
        self._logger.register_key('Misc/RewUpdate')
        self._logger.register_key('Misc/CostUpdate')

    def _adv_lagrange(self):
        return None

    def _train_state(self) -> dict:
        return {**super()._train_state(), 'rew_update': self._rew_update, 'cost_update': self._cost_update}

    def _load_train_state(self, state: dict) -> None:
        super()._load_train_state(state)
        self._rew_update, self._cost_update = int(state['rew_update']), int(state['cost_update'])

    def _surrogate_kind(self) -> int:
        a = self._cfgs.algo_cfgs
        jc = self._window_means()[1]
        if jc <= a.cost_limit + a.distance:
            self._rew_update += 1
            return LOSS_RATIO
        self._cost_update += 1
        return LOSS_COST

    def _log_extra(self) -> None:
        super()._log_extra()
        self._logger.store({'Misc/RewUpdate': self._rew_update, 'Misc/CostUpdate': self._cost_update})


class _SauteMixin:
    """saute/ppo_saute.py:L43-83, saute/trpo_saute.py: the Saute adapter instead of the plain one + Metrics/EpBudget."""

    _adapter_cls = SauteAdapter

    def _init_env(self) -> None:
        _require_synthetic(self._env_id, type(self).__name__)
        t, a = self._cfgs.train_cfgs, self._cfgs.algo_cfgs
        rank = distributed.get_rank()
        self._env = self._adapter_cls(self._env_id, t.vector_env_nums, self._seed, self._cfgs, device=self._device,
                                      env_id_offset=rank * t.vector_env_nums)
        self._steps_per_epoch = distributed.local_steps(a.steps_per_epoch, t.vector_env_nums)

    def _init_log(self) -> None:
        super()._init_log()
        self._logger.register_key('Metrics/EpBudget')

    def _log_epoch(self, epoch, start, epoch_time, roll):
        self._logger.store({'Metrics/EpBudget': self._env.ep_budget_mean()})
        return super()._log_epoch(epoch, start, epoch_time, roll)


class _SimmerMixin(_SauteMixin):
    """simmer/ppo_simmer_pid.py:L48-95: the budget controller acts on the windowed mean episode cost before every update."""

    _adapter_cls = SimmerAdapter

    def _update(self) -> None:
        ws = self._env.window_sums.tolist()                    # {sum EpRet, sum EpCost, sum EpLen, count}, all ranks
        self._env.control_budget(ws[1] / ws[3] if ws[3] > 0 else 0.0)
        super()._update()


@registry.register
class PPOSaute(_SauteMixin, PPO):
    """saute/ppo_saute.py:L28-83."""


@registry.register
class TRPOSaute(_SauteMixin, TRPO):
    """saute/trpo_saute.py."""


@registry.register
class PPOSimmerPID(_SimmerMixin, PPO):
    """simmer/ppo_simmer_pid.py:L30-95."""


@registry.register
class TRPOSimmerPID(_SimmerMixin, TRPO):
    """simmer/trpo_simmer_pid.py."""


class _EarlyTerminatedMixin:
    """early_terminated/ppo_early_terminated.py:L43-66, early_terminated/trpo_early_terminated.py.  The cost-limit rule
    runs in the fused rollout on the synthetic env and in the observe kernel on a registered one."""

    def _init_env(self) -> None:
        t, a = self._cfgs.train_cfgs, self._cfgs.algo_cfgs
        rank = distributed.get_rank()
        cls = EarlyTerminatedAdapter if self._env_id in synthetic_envs() else ExternalEarlyTerminatedAdapter
        self._env = cls(self._env_id, t.vector_env_nums, self._seed, self._cfgs, device=self._device,
                        env_id_offset=rank * t.vector_env_nums)
        self._steps_per_epoch = distributed.local_steps(a.steps_per_epoch, t.vector_env_nums)


@registry.register
class PPOEarlyTerminated(_EarlyTerminatedMixin, PPO):
    """early_terminated/ppo_early_terminated.py:L28-66."""


@registry.register
class TRPOEarlyTerminated(_EarlyTerminatedMixin, TRPO):
    """early_terminated/trpo_early_terminated.py."""


ON_POLICY = ['PolicyGradient', 'PPO', 'PPOLag', 'PDO', 'IPO', 'P3O', 'NaturalPG', 'RCPO', 'TRPO', 'TRPOLag', 'CPO', 'PCPO',
             'FOCOPS', 'CPPOPID', 'TRPOPID', 'OnCRPO', 'PPOSaute', 'TRPOSaute', 'PPOSimmerPID', 'TRPOSimmerPID',
             'PPOEarlyTerminated', 'TRPOEarlyTerminated']
