"""The WideBox test CMDP of tests/external_envs.py as an evaluation sees it: the Evaluator never calls set_seed, so this
variant builds its dynamics with the default seed 0 at the first reset.  Registered under its own id by
tests/golden/make_golden_evaluate.py (reference registry) and tests/test_evaluate_gpu.py (omnisafe_b200 registry)."""
from __future__ import annotations

import external_envs as xe

WIDE_BOX_EVAL_ID = 'WideBoxEval-v0'


def wide_box_eval_cmdp(CMDP, Box):
    base = xe.wide_box_cmdp(CMDP, Box)

    class WideBoxEval(base):
        _support_envs = [WIDE_BOX_EVAL_ID]  # noqa: RUF012

        def reset(self, seed=None, options=None):
            if self._core is None:
                self.set_seed(0)
            return super().reset(seed=seed, options=options)

    return WideBoxEval


def register(CMDP, Box, env_register, registered_ids):
    if WIDE_BOX_EVAL_ID not in registered_ids:
        env_register(wide_box_eval_cmdp(CMDP, Box))
