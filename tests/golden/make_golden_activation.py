"""Golden fixtures of the hidden activations other than tanh: the UNMODIFIED reference (through oracle/ref_shim.py, like
make_golden.py) with actor hidden_sizes [24, 40] and critic hidden_sizes [8, 64] on the synthetic env, once per entry of
CASES (model_cfgs.actor.activation, model_cfgs.critic.activation).

    python tests/golden/make_golden_activation.py

Writes, per case `tag`, with make_golden.py's generators and seeds (as make_golden_hidden.py does for tanh):
- rollout_ppolag_act_<tag>.npz: one rollout epoch (slabs, normaliser, window) from the initial `_flat_theta`;
- update_ppolag_act_<tag>.npz: PPOLag._update on that rollout (initial / final `_flat_theta`, orders, logged losses);
- update_cpo_act_<tag>.npz: CPO's Fisher-vector product, CG solve and one `_update` (line search);
- evaluate_actor_act_<tag>.npz: the library's CPU-initialised actor (`actor_state_dict()`, what epoch-k.pt holds as
  'pi') loaded into the reference's GaussianLearningActor with the case's activation, and that actor's mean on fixed
  rows.
Every file also holds `actor_activation` / `critic_activation`.  Every `theta` is in the reference's flat order; the
tests map it into the kernel layout through omnisafe_b200.models.ParamMap.
"""
from __future__ import annotations

import os
import shutil
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402  (installs the shim, registers the synthetic env with the reference)

ACTOR_HIDDEN, CRITIC_HIDDEN = [24, 40], [8, 64]
# tag -> (actor activation, critic activation); 'softplus' gives the actor and the critics different activations
CASES = {'identity': ('identity', 'identity'), 'relu': ('relu', 'relu'), 'sigmoid': ('sigmoid', 'sigmoid'),
         'softplus': ('softplus', 'relu')}
EVAL_SEED, EVAL_O, EVAL_A = 3, 12, 3


def _set_defaults(actor_act, critic_act):
    """The reference's default config loader, returning configs with the narrow widths and the case's activations."""
    import omnisafe.utils.config as rc

    orig = getattr(rc, '_golden_orig_loader', None) or rc.get_default_kwargs_yaml
    rc._golden_orig_loader = orig

    def load(*args, **kwargs):
        cfgs = orig(*args, **kwargs)
        cfgs.model_cfgs.actor.hidden_sizes = list(ACTOR_HIDDEN)
        cfgs.model_cfgs.critic.hidden_sizes = list(CRITIC_HIDDEN)
        cfgs.model_cfgs.actor.activation = actor_act
        cfgs.model_cfgs.critic.activation = critic_act
        return cfgs

    rc.get_default_kwargs_yaml = load


def gen_evaluate_actor(out_dir, tag, actor_act, critic_act):
    from types import SimpleNamespace as NS

    from gymnasium.spaces import Box
    from omnisafe.models.actor.gaussian_learning_actor import GaussianLearningActor

    from omnisafe_b200.models import ConstraintActorCritic

    mc = NS(actor=NS(hidden_sizes=ACTOR_HIDDEN, activation=actor_act, lr=3e-4),
            critic=NS(hidden_sizes=CRITIC_HIDDEN, activation=critic_act, lr=3e-4),
            actor_type='gaussian_learning', linear_lr_decay=False, weight_initialization_mode='kaiming_uniform')
    model = ConstraintActorCritic(EVAL_O, EVAL_A, mc, epochs=1, device='cpu',
                                  generator=torch.Generator().manual_seed(EVAL_SEED))
    pi = model.actor_state_dict()
    ref = GaussianLearningActor(Box(-10.0, 10.0, (EVAL_O,)), Box(-1.0, 1.0, (EVAL_A,)), ACTOR_HIDDEN, actor_act)
    ref.load_state_dict(pi, strict=True)
    obs = torch.randn(64, EVAL_O, generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        mean = ref.predict(obs, deterministic=True)
    np.savez(os.path.join(out_dir, f'evaluate_actor_act_{tag}.npz'), seed=EVAL_SEED, O=EVAL_O, A=EVAL_A,
             actor_hidden=ACTOR_HIDDEN, critic_hidden=CRITIC_HIDDEN, actor_activation=actor_act,
             critic_activation=critic_act, obs=obs.numpy(), mean=mean.numpy(),
             **{'pi_' + k: v.numpy() for k, v in pi.items()})


def main():
    torch.set_num_threads(1)
    out = mg.OUT
    for tag, (actor_act, critic_act) in CASES.items():
        _set_defaults(actor_act, critic_act)
        tmp = tempfile.mkdtemp()
        mg.OUT = tmp
        try:
            algo = mg.gen_rollout()
            mg.gen_update_ppolag(algo)
            mg.gen_cpo()
        finally:
            mg.OUT = out
        for name in ('rollout_ppolag', 'update_ppolag', 'update_cpo'):
            g = dict(np.load(os.path.join(tmp, f'{name}.npz')))
            np.savez(os.path.join(out, f'{name}_act_{tag}.npz'), actor_hidden=ACTOR_HIDDEN, critic_hidden=CRITIC_HIDDEN,
                     actor_activation=actor_act, critic_activation=critic_act, **g)
        shutil.rmtree(tmp)
        gen_evaluate_actor(out, tag, actor_act, critic_act)
    print('activation golden fixtures written to', out)


if __name__ == '__main__':
    main()
