"""CPU: the parts of the drop-in contract (INTEGRATION.md) that upstream OmniSafe code relies on, checked against what the
unmodified upstream package exposes, stored in tests/golden/upstream_contract.json: the algorithm constructor and
Lagrange.update_lagrange_multiplier parameter lists, and the checkpoint a saved run leaves for the upstream Evaluator
(the keys it reads, the actor state_dict it loads into its own GaussianLearningActor, the Normalizer state_dict)."""
import glob
import inspect
import json
import os

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
with open(os.path.join(ROOT, 'tests', 'golden', 'upstream_contract.json')) as fh:
    UP = json.load(fh)


def test_constructor_and_lagrange_signatures():
    from omnisafe_b200.algorithms import on_policy as mine
    from omnisafe_b200.common.lagrange import Lagrange

    for name in ('PPOLag', 'CPO', 'TRPOLag', 'FOCOPS'):
        assert list(inspect.signature(getattr(mine, name).__init__).parameters)[1:] == UP['algo_init_params'], name
    assert list(inspect.signature(Lagrange.update_lagrange_multiplier).parameters) == UP['lagrange_update_params']


def test_checkpoint_matches_what_the_upstream_evaluator_loads(tmp_path):
    from omnisafe_b200.common.logger import Logger
    from omnisafe_b200.common.normalizer import Normalizer
    from omnisafe_b200.models import ConstraintActorCritic
    from omnisafe_b200.utils.config import get_default_kwargs_yaml

    O, A = UP['obs_dim'], UP['act_dim']
    cfgs = get_default_kwargs_yaml('PPOLag', 'SyntheticBox-v0', 'on-policy')
    cfgs.recurisve_update({'exp_name': 'PPOLag-{SyntheticBox-v0}', 'env_id': 'SyntheticBox-v0', 'algo': 'PPOLag',
                           'env_cfgs': {'obs_dim': O, 'act_dim': A, 'max_episode_steps': 8, 'term_prob': 0.0},
                           'logger_cfgs': {'log_dir': str(tmp_path)}, 'train_cfgs': {'epochs': 1}})
    ac = ConstraintActorCritic(O, A, cfgs.model_cfgs, epochs=1, device='cpu')
    norm = Normalizer((O,), clip=5.0, device='cpu')
    logger = Logger(str(tmp_path), cfgs.exp_name, seed=0, config=cfgs)
    logger.setup_torch_saver({'pi': ac.actor_state_dict, 'obs_normalizer': norm})
    logger.torch_save()
    logger.close()
    (path,) = glob.glob(os.path.join(logger.log_dir, 'torch_save', 'epoch-0.pt'))
    params = torch.load(path, weights_only=False)
    assert set(UP['checkpoint_keys_read_by_evaluator']) <= set(params)
    assert {k: list(v.shape) for k, v in params['pi'].items()} == UP['actor_state_dict']
    assert {k: list(v.shape) for k, v in params['obs_normalizer'].items()} == UP['obs_normalizer_state_dict']
