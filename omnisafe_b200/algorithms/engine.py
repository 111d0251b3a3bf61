"""Device workspace + thin call wrappers for the learner kernels (the "operator boundary" between
the algorithm classes and the C ABI).  Every method launches asynchronously on the current stream;
only the `*_item` helpers synchronise (they are used where the reference itself calls `.item()`).
"""
from __future__ import annotations

import torch

from omnisafe_b200._lib import current_stream, lib, ptr
from omnisafe_b200.algorithms.torch_loss import feistel_order
from omnisafe_b200.utils import distributed
from omnisafe_b200.utils.train_state import restore, snapshot

LOSS_PPO_CLIP, LOSS_RATIO, LOSS_FOCOPS, LOSS_COST, LOSS_P3O = 0, 1, 2, 3, 5
NET_ACTOR, NET_CRITIC_R, NET_CRITIC_C = 1, 2, 4


class UpdateEngine:
    def __init__(self, agent, buf) -> None:
        self.agent, self.buf = agent, buf
        dev = agent.device
        self.O, self.A = agent.obs_dim, agent.act_dim
        self.P = agent.layout['total']
        self.Pa = agent.layout['actor']['size']
        self.total = buf.T * buf.N
        f32 = dict(dtype=torch.float32, device=dev)
        self.gpart = torch.zeros(148 * self.P, **f32)
        self.stats_part = torch.zeros(148 * 3 * 8, **f32)
        self.sumsq_part = torch.zeros(6 * lib().osb_optim_blocks(self.O, self.A), **f32)
        self.train_stats = torch.zeros(3 * 8, **f32)
        self.eval_ws = torch.zeros(296 * 8, dtype=torch.float64, device=dev)
        self.eval_out = torch.zeros(8, dtype=torch.float64, device=dev)
        self.stop_flag = torch.zeros(1, dtype=torch.int32, device=dev)
        self.kl_state = torch.zeros(4, **f32)
        self.mu_old = torch.zeros(buf.T, buf.N, self.A, **f32)
        self.logstd_old = torch.zeros(self.A, **f32)
        # natural-gradient workspace
        self.fvp_part = torch.zeros(148 * self.Pa, **f32)
        self.fvp_dmu = torch.zeros(self.total * self.A, **f32)     # tangent of mu per row (tensor-core FVP)
        self.cg_x = torch.zeros(self.Pa, **f32)
        self.cg_r = torch.zeros(self.Pa, **f32)
        self.cg_p = torch.zeros(self.Pa, **f32)
        self.cg_z = torch.zeros(self.Pa, **f32)
        self.cg_scalars = torch.zeros(4, **f32)
        self.scalar = torch.zeros(4, **f32)
        self._perm_seed = 0x1234567
        self.precision = 0   # 0 = exact fp32 FMA tiles, 1 = TF32 wgmma tiles (5e-3), 2 = split-bf16 wgmma tiles (fp32-level)

    # ---- helpers ----------------------------------------------------------------------------
    def _tc(self) -> bool:
        return self.precision == 1 and self.O <= 512      # obs dims > 64: layer 1 K-chunked (rollout stays on fp32 tiles)

    def _x3(self) -> bool:
        return self.precision == 2 and self.O <= 64        # split-bf16 tiles: fp32-level results on the tensor cores

    def _eval_fn(self):
        if self._x3():
            return lib().osb_actor_eval_x3
        return lib().osb_actor_eval_tc if self._tc() else lib().osb_actor_eval

    def _batch_ptrs(self):
        d = self.buf.data
        return [ptr(d['obs']), ptr(d['act']), ptr(d['logp']), ptr(d['adv_r']), ptr(d['adv_c']),
                ptr(d['target_value_r']), ptr(d['target_value_c'])]

    def next_perm_seed(self) -> int:
        self._perm_seed = (self._perm_seed * 1664525 + 1013904223) & 0xFFFFFFFF
        return self._perm_seed

    def train_state(self) -> dict:
        """The minibatch-permutation LCG and kl_state: NaturalPG / RCPO log the KL an epoch leaves in kl_state[0] as the
        next epoch's final KL (NaturalPG._update).  Everything else here is rewritten before it is read in an epoch."""
        return {'perm_seed': self._perm_seed, 'kl_state': snapshot(self.kl_state)[0]}

    def load_train_state(self, state: dict) -> None:
        self._perm_seed = int(state['perm_seed'])
        restore(self.kl_state, state['kl_state'], 'update kl_state')

    # ---- PolicyGradient._update loop (one C call) -----------------------------------------
    def ppo_epoch(self, *, loss_kind, lagrange, net_mask, batch_size, update_iters, clip=0.2,
                  entropy_coef=0.0, focops_lam=1.0, focops_eta=0.0, critic_norm_coef=0.0,
                  max_grad_norm=0.0, lr_actor=0.0, lr_critic=0.0, target_kl=0.0, kl_early_stop=False,
                  perm=None, precision: int | None = None) -> None:
        a = self.agent
        a.apply_net_spec()
        if perm is not None:
            assert perm.dtype == torch.int32 and perm.shape == (update_iters, self.total)
        lib().osb_ppo_update_epoch(
            ptr(a.theta), ptr(a.grad), ptr(a.adam_m), ptr(a.adam_v), ptr(a.adam_step), self.O, self.A,
            *self._batch_ptrs(), ptr(self.mu_old), ptr(self.logstd_old), ptr(self.buf.adv_moments),
            ptr(perm), self.total, self.next_perm_seed(), int(batch_size), int(update_iters),
            int(loss_kind), float(clip), float(entropy_coef), float(focops_lam), float(focops_eta),
            ptr(lagrange), int(net_mask), float(critic_norm_coef), float(max_grad_norm),
            float(lr_actor), float(lr_critic), float(target_kl), int(kl_early_stop),
            ptr(self.gpart), ptr(self.stats_part), ptr(self.sumsq_part), ptr(self.train_stats),
            ptr(self.eval_ws), ptr(self.eval_out), ptr(self.stop_flag), ptr(self.kl_state),
            self.precision if precision is None else int(precision),
            distributed.nccl_comm(), distributed.world_size(), *distributed.p2p_exchange(self.P)[:2],
            distributed.get_rank(), distributed.p2p_exchange(self.P)[2], current_stream())

    # ---- PolicyGradient._update with objectives in PyTorch ---------------------------------
    def _optim_step(self, gpart, stats_part, nb, net_mask, critic_norm_coef, max_grad_norm, lr_actor, lr_critic):
        """Reduce the partials, clip, average over ranks and Adam-step the networks of `net_mask` (the order of
        osb_ppo_update_epoch)."""
        a, s, w = self.agent, current_stream(), distributed.world_size()
        if w == 1:
            lib().osb_optim_fused(ptr(gpart), ptr(stats_part), nb, self.O, self.A, ptr(a.theta), ptr(a.grad),
                                  ptr(a.adam_m), ptr(a.adam_v), ptr(a.adam_step), float(critic_norm_coef),
                                  float(max_grad_norm), float(lr_actor), float(lr_critic), float(lr_critic), net_mask,
                                  ptr(self.sumsq_part), ptr(self.train_stats), ptr(self.stop_flag), s)
            return
        lib().osb_grad_reduce(ptr(gpart), ptr(stats_part), nb, self.O, self.A, ptr(a.theta), ptr(a.grad),
                              float(critic_norm_coef), net_mask, ptr(self.sumsq_part), ptr(a.adam_step),
                              ptr(self.train_stats), ptr(self.stop_flag), s)
        for do_clip, do_adam, scale in ((1, 0, 1.0), (0, 1, 1.0 / w)):
            if do_adam:
                distributed.all_reduce_(a.grad)
            lib().osb_clip_adam(ptr(a.grad), ptr(a.theta), ptr(a.adam_m), ptr(a.adam_v), ptr(a.adam_step),
                                ptr(self.sumsq_part), self.O, self.A, float(max_grad_norm), float(lr_actor),
                                float(lr_critic), float(lr_critic), float(scale), float(critic_norm_coef),
                                ptr(self.train_stats), do_clip, do_adam, net_mask, ptr(self.stop_flag), s)

    def adam_step(self, net: int, grad: torch.Tensor, lr: float) -> None:
        """torch.optim.Adam.step() of critic `net` (1 reward, 2 cost) on `grad`, its flat gradient as its optimiser
        holds it (clipped and rank-averaged by the caller, or not): the kernels' Adam on that network's slice of theta,
        with its step count and `lr`.  Nothing is clipped, averaged or added here."""
        a, s = self.agent, current_stream()
        if not hasattr(self, 'hook_gpart'):
            self.hook_gpart = torch.zeros(self.P, dtype=torch.float32, device=a.device)
            self.hook_stats = torch.zeros(3 * 8, dtype=torch.float32, device=a.device)
        lay = a.layout['reward_critic' if net == 1 else 'cost_critic']
        self.hook_gpart[lay['start']:lay['start'] + lay['size']].copy_(grad)
        self.hook_stats.zero_()
        self.hook_stats[8 * net + 3] = 1.0
        lib().osb_grad_reduce(ptr(self.hook_gpart), ptr(self.hook_stats), 1, self.O, self.A, ptr(a.theta), ptr(a.grad),
                              0.0, 1 << net, ptr(self.sumsq_part), ptr(a.adam_step), ptr(self.train_stats), 0, s)
        lib().osb_clip_adam(ptr(a.grad), ptr(a.theta), ptr(a.adam_m), ptr(a.adam_v), ptr(a.adam_step),
                            ptr(self.sumsq_part), self.O, self.A, 0.0, 0.0, float(lr), float(lr), 1.0, 0.0,
                            ptr(self.train_stats), 0, 1, 1 << net, 0, s)

    def stepwise_epoch(self, steps: dict, *, loss_kind, lagrange, net_mask, batch_size, update_iters, clip=0.2,
                       entropy_coef=0.0, focops_lam=1.0, focops_eta=0.0, critic_norm_coef=0.0, max_grad_norm=0.0,
                       lr_actor=0.0, lr_critic=0.0, target_kl=0.0, kl_early_stop=False, perm=None) -> None:
        """ppo_epoch as a host loop of minibatch steps, with networks trained through autograd.  Per minibatch of the
        sample order the kernels draw (or `perm`), the networks of `net_mask` step in the reference's order: reward
        critic, cost critic, actor.  A network with a callable in `steps` (net bit -> callable(rows), rows the slab
        rows [count] int64) runs it; the others take the stepwise kernel step (osb_minibatch_grad* + the optimiser),
        consecutive ones in one launch.  The actor's callable returns (loss, gradient of the actor parameters), which
        the kernels clip, rank-average and Adam-step; a critic's callable trains its network itself.  When the actor
        trains, the old policy is snapshotted first and the full-batch KL check runs after each pass, as in ppo_epoch."""
        a, s = self.agent, current_stream()
        a.apply_net_spec()
        if perm is not None:
            assert perm.dtype == torch.int32 and perm.shape == (update_iters, self.total)
        self.stop_flag.zero_()
        self.kl_state.zero_()
        self.train_stats.zero_()
        train_actor = bool(net_mask & NET_ACTOR)
        if train_actor:
            self.snapshot_old_policy()
        if not hasattr(self, 'actor_gpart'):
            self.actor_gpart = torch.zeros(self.P, dtype=torch.float32, device=a.device)
            self.actor_stats = torch.zeros(3 * 8, dtype=torch.float32, device=a.device)
        seed = self.next_perm_seed()
        opt = dict(critic_norm_coef=critic_norm_coef, max_grad_norm=max_grad_norm, lr_actor=lr_actor,
                   lr_critic=lr_critic)
        tiles = self._tc() or self._x3()
        grad_fn = lib().osb_minibatch_grad_x3 if self._x3() else (lib().osb_minibatch_grad_tc if self._tc()
                                                                   else lib().osb_minibatch_grad)

        def kernel_step(mask, order, start, count):
            loss = ((int(loss_kind), float(clip), float(entropy_coef), float(focops_lam), float(focops_eta),
                     ptr(lagrange)) if mask & NET_ACTOR else (LOSS_RATIO, 0.0, 0.0, 1.0, 0.0, 0))
            grad_fn(ptr(a.theta), self.O, self.A, *self._batch_ptrs(), ptr(self.mu_old), ptr(self.buf.adv_moments),
                    ptr(order), self.total, 0, start, count, *loss, ptr(self.logstd_old), mask, ptr(self.gpart),
                    ptr(self.stats_part), ptr(self.stop_flag), s)
            nb = lib().osb_tc_grid_blocks(count, mask) if tiles else lib().osb_update_grid_blocks(count)
            self._optim_step(self.gpart, self.stats_part, nb, mask, **opt)

        for it in range(update_iters):
            if perm is not None:
                order = perm[it].contiguous()
            else:
                it_seed = (seed + 0x9E3779B9 * it) & 0xFFFFFFFF
                order = feistel_order(self.total, it_seed, a.device).to(torch.int32)
            rows_all = order.to(torch.int64)
            for start in range(0, self.total, batch_size):
                count = min(batch_size, self.total - start)
                rows = rows_all[start:start + count]
                pending = 0
                for bit in (NET_CRITIC_R, NET_CRITIC_C, NET_ACTOR):
                    if not net_mask & bit:
                        continue
                    if bit not in steps:
                        pending |= bit
                        continue
                    if pending:
                        kernel_step(pending, order, start, count)
                        pending = 0
                    if bit != NET_ACTOR:
                        steps[bit](rows)
                        continue
                    loss, grad = steps[bit](rows)
                    self.actor_gpart[: self.Pa].copy_(grad)
                    self.actor_stats[0] = loss.detach()
                    self.actor_stats[3] = 1.0
                    self._optim_step(self.actor_gpart, self.actor_stats, 1, NET_ACTOR, **opt)
                if pending:
                    kernel_step(pending, order, start, count)
            if not train_actor:
                continue
            d = self.buf.data
            self._eval_fn()(ptr(a.theta), self.O, self.A, ptr(d['obs']), ptr(d['act']), ptr(d['logp']),
                            ptr(d['adv_r']), ptr(d['adv_c']), ptr(self.mu_old), ptr(self.logstd_old),
                            ptr(self.buf.adv_moments), ptr(lagrange), self.total, 1, 0, ptr(self.eval_ws),
                            ptr(self.eval_out), s)
            if distributed.world_size() > 1:
                distributed.all_reduce_(self.eval_out)
            lib().osb_kl_check(ptr(self.eval_out), float(target_kl), int(kl_early_stop), ptr(self.stop_flag),
                               ptr(self.kl_state), s)
            if kl_early_stop and it + 1 < update_iters and int(self.stop_flag.item()):
                break

    # ---- full-batch pieces for the natural-gradient family ---------------------------------
    def snapshot_old_policy(self) -> None:
        """p_dist = actor(obs) at the current parameters (trpo.py:L177, cpo.py:L366)."""
        a = self.agent
        a.apply_net_spec()
        self._eval_fn()(ptr(a.theta), self.O, self.A, ptr(self.buf.data['obs']), 0, 0, 0, 0, 0, 0,
                        0, 0, self.total, 1, ptr(self.mu_old), 0, 0, current_stream())
        self.logstd_old.copy_(a.theta[:self.A])

    def actor_loss_grad(self, loss_kind, lagrange, out_grad: torch.Tensor, sign: float = 1.0) -> torch.Tensor:
        """loss.backward() of the full-batch surrogate + avg_grads (natural_pg.py:L150-157):
        out_grad <- sign * d loss / d theta_actor; returns the device scalar `loss` (rank-averaged)."""
        a = self.agent
        a.apply_net_spec()
        if (self._tc() or self._x3()) and loss_kind in (LOSS_RATIO, LOSS_COST):
            nb = lib().osb_tc_grid_blocks(self.total, NET_ACTOR)
            (lib().osb_minibatch_grad_x3 if self._x3() else lib().osb_minibatch_grad_tc)(
                ptr(a.theta), self.O, self.A, *self._batch_ptrs(), ptr(self.mu_old), ptr(self.buf.adv_moments),
                0, self.total, self.next_perm_seed(), 0, self.total, int(loss_kind), 0.0, 0.0, 1.0, 0.0,
                ptr(lagrange), ptr(self.logstd_old), NET_ACTOR, ptr(self.gpart), ptr(self.stats_part), 0,
                current_stream())
        else:
            nb = lib().osb_update_grid_blocks(self.total)
            lib().osb_minibatch_grad(
                ptr(a.theta), self.O, self.A, *self._batch_ptrs(), ptr(self.mu_old),
                ptr(self.buf.adv_moments), 0, self.total, 0, 0, self.total, int(loss_kind), 0.0, 0.0, 1.0,
                0.0, ptr(lagrange), ptr(self.logstd_old), NET_ACTOR, ptr(self.gpart),
                ptr(self.stats_part), 0, current_stream())
        w = distributed.world_size()
        lib().osb_reduce_partials(ptr(self.gpart), nb, self.P, self.Pa, sign / w, 0, 0.0, ptr(out_grad),
                                  current_stream())
        st = self.stats_part[: nb * 24].view(nb, 3, 8)[:, 0, :].sum(0)
        loss = (st[0] / st[3]).reshape(1) / w
        if w > 1:
            distributed.all_reduce_(out_grad)
            distributed.all_reduce_(loss)
        return loss

    def fvp(self, vec: torch.Tensor, out: torch.Tensor, damping: float, stride: int = 1) -> None:
        """NaturalPG._fvp (natural_pg.py:L74-119): out <- avg_ranks(F vec) + damping * vec."""
        a = self.agent
        a.apply_net_spec()
        if self._x3():
            nb = lib().osb_tc_grid_blocks((self.total + stride - 1) // stride, NET_ACTOR)
            lib().osb_fvp_partials_x3(ptr(a.theta), ptr(vec), self.O, self.A, ptr(self.buf.data['obs']),
                                      self.total, stride, ptr(self.fvp_dmu), ptr(self.fvp_part),
                                      ptr(self.stats_part), current_stream())
        elif self._tc():
            nb = lib().osb_tc_grid_blocks((self.total + stride - 1) // stride, NET_ACTOR)
            lib().osb_fvp_partials_tc(ptr(a.theta), ptr(vec), self.O, self.A, ptr(self.buf.data['obs']),
                                      self.total, stride, ptr(self.fvp_dmu), ptr(self.fvp_part),
                                      ptr(self.stats_part), current_stream())
        else:
            nb = lib().osb_fvp_grid_blocks(self.total, stride)
            lib().osb_fvp_partials(ptr(a.theta), ptr(vec), self.O, self.A, ptr(self.buf.data['obs']),
                                   self.total, stride, ptr(self.fvp_part), current_stream())
        w = distributed.world_size()
        if w == 1:
            lib().osb_reduce_partials(ptr(self.fvp_part), nb, self.Pa, self.Pa, 1.0, ptr(vec), float(damping),
                                      ptr(out), current_stream())
        else:
            lib().osb_reduce_partials(ptr(self.fvp_part), nb, self.Pa, self.Pa, 1.0 / w, 0, 0.0, ptr(out),
                                      current_stream())
            distributed.all_reduce_(out)
            out.add_(vec, alpha=float(damping))

    def conjugate_gradients(self, b: torch.Tensor, num_steps: int, damping: float, stride: int = 1,
                            residual_tol: float = 1e-10, eps: float = 1e-6) -> torch.Tensor:
        """utils/math.py:L86-132 with device-resident state; returns a fresh tensor x."""
        s = current_stream()
        lib().osb_cg_init(ptr(b), self.Pa, ptr(self.cg_x), ptr(self.cg_r), ptr(self.cg_p),
                          ptr(self.cg_scalars), s)
        for _ in range(num_steps):
            self.fvp(self.cg_p, self.cg_z, damping, stride)
            lib().osb_cg_step(ptr(self.cg_z), self.Pa, ptr(self.cg_x), ptr(self.cg_r), ptr(self.cg_p),
                              ptr(self.cg_scalars), float(residual_tol), float(eps), s)
        return self.cg_x.clone()

    def dot(self, a: torch.Tensor, b: torch.Tensor) -> float:
        lib().osb_dot(ptr(a), ptr(b), a.numel(), ptr(self.scalar), current_stream())
        return float(self.scalar[0].item())

    def evaluate(self, theta_actor: torch.Tensor, lagrange) -> dict:
        """Surrogates and KL of a trial actor (line searches trpo.py:L102-138, cpo.py:L114-171).
        Returns python floats averaged over ranks: loss (= -mean ratio*adv), loss_r (= -mean
        ratio*adv_r), loss_c (= mean ratio*adv_c), kl (= mean over samples AND action dims)."""
        d = self.buf.data
        self.agent.apply_net_spec()
        self._eval_fn()(ptr(theta_actor), self.O, self.A, ptr(d['obs']), ptr(d['act']), ptr(d['logp']),
                        ptr(d['adv_r']), ptr(d['adv_c']), ptr(self.mu_old), ptr(self.logstd_old),
                        ptr(self.buf.adv_moments), ptr(lagrange), self.total, 1, 0, ptr(self.eval_ws),
                        ptr(self.eval_out), current_stream())
        if distributed.world_size() > 1:
            distributed.all_reduce_(self.eval_out)
        o = self.eval_out.tolist()
        n = o[4]
        return {'kl': o[0] / (n * self.A), 'kl_sum': o[0] / n, 'loss': -o[1] / n, 'loss_c': o[2] / n,
                'ratio': o[3] / n, 'loss_r': -o[5] / n}
