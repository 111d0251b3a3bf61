"""omnisafe_b200: H100-native (sm_90a) on-policy SafeRL hot path behind the omnisafe surface."""
from omnisafe_b200.algorithms import ALGORITHMS  # noqa: F401
from omnisafe_b200.algorithms.algo_wrapper import AlgoWrapper as Agent  # noqa: F401
from omnisafe_b200.evaluator import Evaluator  # noqa: F401

__version__ = '0.1.0'
