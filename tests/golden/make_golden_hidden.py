"""Golden fixtures of networks narrower than 64: the UNMODIFIED reference (through oracle/ref_shim.py, like
make_golden.py) with actor hidden_sizes [24, 40] and critic hidden_sizes [8, 64] on the synthetic env.

    python tests/golden/make_golden_hidden.py

Writes, with make_golden.py's generators and seeds:
- rollout_ppolag_hidden.npz: one rollout epoch (slabs, normaliser, window) from the initial `_flat_theta`;
- update_ppolag_hidden.npz: PPOLag._update on that rollout (initial / final `_flat_theta`, orders, logged losses);
- update_cpo_hidden.npz: CPO's Fisher-vector product, CG solve and one `_update` (line search);
- evaluate_actor_hidden.npz: the library's CPU-initialised actor of those widths (`actor_state_dict()`, what
  epoch-k.pt holds as 'pi') loaded into the reference's GaussianLearningActor, and that actor's mean on fixed rows.
Every `theta` is in the reference's flat order (named_parameters of actor, reward critic, cost critic); the tests map
it into the kernel layout through omnisafe_b200.models.ParamMap.
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
EVAL_SEED, EVAL_O, EVAL_A = 3, 12, 3


def _narrow_defaults():
    """The reference's default config loader, returning configs with the narrow widths."""
    import omnisafe.utils.config as rc

    orig = rc.get_default_kwargs_yaml

    def load(*args, **kwargs):
        cfgs = orig(*args, **kwargs)
        cfgs.model_cfgs.actor.hidden_sizes = list(ACTOR_HIDDEN)
        cfgs.model_cfgs.critic.hidden_sizes = list(CRITIC_HIDDEN)
        return cfgs

    rc.get_default_kwargs_yaml = load


def gen_evaluate_actor(out_dir):
    from types import SimpleNamespace as NS

    from gymnasium.spaces import Box
    from omnisafe.models.actor.gaussian_learning_actor import GaussianLearningActor

    from omnisafe_b200.models import ConstraintActorCritic

    def net(hs):
        return NS(hidden_sizes=hs, activation='tanh', lr=3e-4)

    mc = NS(actor=net(ACTOR_HIDDEN), critic=net(CRITIC_HIDDEN), actor_type='gaussian_learning', linear_lr_decay=False,
            weight_initialization_mode='kaiming_uniform')
    model = ConstraintActorCritic(EVAL_O, EVAL_A, mc, epochs=1, device='cpu',
                                  generator=torch.Generator().manual_seed(EVAL_SEED))
    pi = model.actor_state_dict()
    ref = GaussianLearningActor(Box(-10.0, 10.0, (EVAL_O,)), Box(-1.0, 1.0, (EVAL_A,)), ACTOR_HIDDEN, 'tanh')
    ref.load_state_dict(pi, strict=True)
    obs = torch.randn(64, EVAL_O, generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        mean = ref.predict(obs, deterministic=True)
    np.savez(os.path.join(out_dir, 'evaluate_actor_hidden.npz'), seed=EVAL_SEED, O=EVAL_O, A=EVAL_A,
             actor_hidden=ACTOR_HIDDEN, critic_hidden=CRITIC_HIDDEN, obs=obs.numpy(), mean=mean.numpy(),
             **{'pi_' + k: v.numpy() for k, v in pi.items()})


def main():
    torch.set_num_threads(1)
    _narrow_defaults()
    tmp = tempfile.mkdtemp()
    out, mg.OUT = mg.OUT, tmp
    try:
        algo = mg.gen_rollout()
        mg.gen_update_ppolag(algo)
        mg.gen_cpo()
    finally:
        mg.OUT = out
    for name in ('rollout_ppolag', 'update_ppolag', 'update_cpo'):
        g = dict(np.load(os.path.join(tmp, f'{name}.npz')))
        np.savez(os.path.join(out, f'{name}_hidden.npz'), actor_hidden=ACTOR_HIDDEN, critic_hidden=CRITIC_HIDDEN, **g)
    shutil.rmtree(tmp)
    gen_evaluate_actor(out)
    print('hidden-width golden fixtures written to', out)


if __name__ == '__main__':
    main()
