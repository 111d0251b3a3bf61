"""Worker of the EarlyTerminated resume tests (tests/test_external_early_gpu.py): tests/resume_worker.py with the
graph-safe WideBox that has the per-env reset hook and the state hooks registered as well.

    python tests/early_resume_worker.py resume <state_dir> <out.json> <save_state_freq>
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'tests')):
    if p not in sys.path:
        sys.path.insert(0, p)

import early_envs as ee  # noqa: E402
import resume_worker as rw  # noqa: E402

GRAPH_RESET_ID = 'ResumableGraphWideBoxReset-v0'


def register_envs() -> None:
    from omnisafe_b200.envs import CMDP, ENV_REGISTRY, Box, env_register

    rw.register_envs()
    if GRAPH_RESET_ID in ENV_REGISTRY.support_envs():
        return
    GraphWideBoxReset = ee.reset_envs_cmdps(CMDP, Box)[-1]

    class ResumableGraphWideBoxReset(rw._with_hooks(GraphWideBoxReset)):
        _support_envs = [GRAPH_RESET_ID]  # noqa: RUF012

    env_register(ResumableGraphWideBoxReset)


if __name__ == '__main__':
    register_envs()
    rw.main(sys.argv[1:])
