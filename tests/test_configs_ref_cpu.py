"""CPU: every shipped YAML `defaults` block equals the upstream block of the same algorithm key for key (plus the
`matmul_precision` extension and the env_cfgs placeholder).  The upstream blocks (omnisafe/configs/on-policy/*.yaml,
flattened to dotted keys) are stored in tests/golden/upstream_config_defaults.json."""
import json
import os

import yaml

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
UPSTREAM = os.path.join(ROOT, 'tests', 'golden', 'upstream_config_defaults.json')
MINE = os.path.join(ROOT, 'omnisafe_b200', 'configs', 'on-policy')


def _flat(d, pre=''):
    out = {}
    for k, v in d.items():
        if isinstance(v, dict):
            out.update(_flat(v, pre + k + '.'))
        else:
            out[pre + k] = v
    return out


def test_yaml_defaults_equal_upstream():
    from omnisafe_b200.algorithms import ALGORITHMS

    with open(UPSTREAM) as fh:
        upstream = json.load(fh)
    names = sorted(f[:-5] for f in os.listdir(MINE) if f.endswith('.yaml'))
    assert set(names) == set(ALGORITHMS['on-policy'])          # one YAML per registered class
    assert set(names) == set(upstream)
    for name in names:
        ref = upstream[name]
        with open(os.path.join(MINE, name + '.yaml')) as fh:
            doc = yaml.safe_load(fh)
        mine = _flat(doc['defaults'])
        assert mine.pop('train_cfgs.matmul_precision') == 'fp32', name        # parity arithmetic by default
        assert mine == ref, (name, {k: (ref.get(k), mine.get(k)) for k in set(ref) | set(mine) if ref.get(k) != mine.get(k)})
        assert 'SyntheticBox-v0' in doc                                           # the synthetic workload block
