"""Environment side of the hot path: the HBM-resident synthetic Box CMDP and user-registered CMDPs."""
from omnisafe_b200.envs.core import (CMDP, ENV_REGISTRY, Box, check_env, env_register, env_unregister,  # noqa: F401
                                     is_registered, make, support_envs)
from omnisafe_b200.envs.synthetic import SyntheticBoxEnv, env_bias  # noqa: F401
