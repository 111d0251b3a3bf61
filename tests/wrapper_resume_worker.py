"""Worker of the wrapper-env resume tests (tests/test_external_wrappers_gpu.py): tests/resume_worker.py with the
graph-safe wrapped box of tests/wrapper_envs.py and the state hooks registered as well.

    python tests/wrapper_resume_worker.py resume <state_dir> <out.json> <save_state_freq>
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'tests')):
    if p not in sys.path:
        sys.path.insert(0, p)

import resume_worker as rw  # noqa: E402
import wrapper_envs as we  # noqa: E402

WRAPPED_RESUME_ID = 'ResumableWrappedBox-v0'
GRAPH_WRAPPED_RESUME_ID = 'ResumableGraphWrappedBoxReset-v0'


def register_envs() -> None:
    from omnisafe_b200.envs import CMDP, ENV_REGISTRY, Box, env_register

    rw.register_envs()
    if GRAPH_WRAPPED_RESUME_ID in ENV_REGISTRY.support_envs():
        return
    classes = we.wrapper_cmdps(CMDP, Box)

    class ResumableWrappedBox(rw._with_hooks(classes[0])):
        _support_envs = [WRAPPED_RESUME_ID]  # noqa: RUF012

    class ResumableGraphWrappedBoxReset(rw._with_hooks(classes[3])):
        _support_envs = [GRAPH_WRAPPED_RESUME_ID]  # noqa: RUF012

    env_register(ResumableWrappedBox)
    env_register(ResumableGraphWrappedBoxReset)


if __name__ == '__main__':
    register_envs()
    rw.main(sys.argv[1:])
