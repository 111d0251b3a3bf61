"""GPU: the policy-step kernel behind ConstraintActorCritic.step / actor / critics (csrc/policy.cu) against reference
modules in fp64, against Normal.rsample under the same seed, against the rollout's slabs, under CUDA-graph replay, and
end to end: acting between epochs leaves training untouched, and a checkpoint's actor acts like the live model."""
import os
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch
from torch.distributions import Normal

import external_envs as xe

pytestmark = pytest.mark.gpu

TOL = {0: 2e-5, 1: 5e-3, 2: 2e-5}     # fp32 / tf32 / bf16x3: the rollout tests' bars


@pytest.fixture(scope='module', autouse=True)
def _registered():
    from omnisafe_b200.envs import CMDP, Box, ENV_REGISTRY, env_register

    xe.register(CMDP, Box, env_register, ENV_REGISTRY.support_envs())


def _model_cfgs():
    net = NS(hidden_sizes=[64, 64], activation='tanh', lr=3e-4)
    return NS(actor=net, critic=net, actor_type='gaussian_learning', linear_lr_decay=True,
              weight_initialization_mode='kaiming_uniform')


def _model(dev, O, A, precision, seed=0):
    from omnisafe_b200.models import ConstraintActorCritic

    m = ConstraintActorCritic(O, A, _model_cfgs(), epochs=1, device=dev, generator=torch.Generator().manual_seed(seed))
    g = torch.Generator().manual_seed(seed + 1)
    m.named_views('actor')['log_std'].copy_(torch.empty(A).uniform_(-1.0, 0.5, generator=g))
    m.precision = precision
    return m


def _reference(m):
    """nn.Sequential actor / critics in fp64 from the live theta, loaded under the reference's key names."""
    dev, O, A = m.device, m.obs_dim, m.act_dim

    def trunk(out):
        return torch.nn.Sequential(torch.nn.Linear(O, 64), torch.nn.Tanh(), torch.nn.Linear(64, 64), torch.nn.Tanh(),
                                   torch.nn.Linear(64, out)).double().to(dev)

    actor = torch.nn.Module()
    actor.mean = trunk(A)
    actor.log_std = torch.nn.Parameter(torch.zeros(A))
    actor.load_state_dict(m.actor_state_dict())
    actor.double().to(dev)
    critics = []
    for net in ('reward_critic', 'cost_critic'):
        c = torch.nn.Module()
        c.critic_0 = trunk(1)
        c.load_state_dict({k: v.double() for k, v in m.named_views(net).items()})
        critics.append(c.critic_0)
    return actor, critics


def _close(got, want, tol, what):
    np.testing.assert_allclose(got.double().cpu().numpy(), want.double().cpu().numpy(), rtol=tol, atol=tol, err_msg=what)


@pytest.mark.parametrize('precision', [0, 1, 2])
@pytest.mark.parametrize('O', [17, 45, 60, 64, 65, 111, 376])
def test_matches_reference_modules(cuda, precision, O):
    tol = TOL[precision]
    for A in (1, 3, 8, 16):
        m = _model(cuda, O, A, precision, seed=O + A)
        actor, (vr_net, vc_net) = _reference(m)
        std64 = torch.exp(actor.log_std.detach())
        for B in ((1, 7, 128, 4097, 65536) if A == 8 else (1, 7, 4097)):
            g = torch.Generator(device=cuda).manual_seed(B)
            obs = torch.randn(B, O, device=cuda, generator=g).clamp_(-5, 5)
            with torch.no_grad():
                mean = actor.mean(obs.double())
                vr, vc = vr_net(obs.double()).squeeze(-1), vc_net(obs.double()).squeeze(-1)
            what = f'precision {precision} O {O} A {A} B {B}'
            act, v_r, v_c, logp = m.step(obs, deterministic=True)
            assert act.shape == (B, A) and v_r.shape == (B,) and v_c.shape == (B,) and logp.shape == (B,)
            _close(act, mean, tol, 'mean ' + what)
            _close(v_r, vr, tol, 'value_r ' + what)
            _close(v_c, vc, tol, 'value_c ' + what)
            _close(logp, Normal(mean, std64).log_prob(mean).sum(-1), tol, 'logp(mean) ' + what)
            assert torch.equal(m.actor.predict(obs, deterministic=True), act)      # deterministic: act == mean
            dist = m.actor.forward(obs)
            assert torch.equal(dist.mean, act)
            x = torch.randn(B, A, device=cuda, generator=g)                          # an arbitrary action
            _close(m.actor.log_prob(x), Normal(mean, std64).log_prob(x.double()).sum(-1), tol, 'log_prob(x) ' + what)
            assert torch.equal(m.reward_critic(obs)[0], v_r) and torch.equal(m.cost_critic(obs)[0], v_c)
    # call shapes: [O] and [..., O]; a CPU tensor is moved to the model's device
    obs = torch.randn(2, 3, O).clamp_(-5, 5)
    act, v_r, v_c, logp = m.step(obs, deterministic=True)
    assert act.shape == (2, 3, A) and v_r.shape == (2, 3) and logp.shape == (2, 3) and act.device == cuda
    one = m.step(obs[1, 2], deterministic=True)
    assert one[0].shape == (A,) and one[1].shape == () and one[3].shape == ()
    assert torch.equal(one[0], act[1, 2]) and torch.equal(one[1], v_r[1, 2]) and torch.equal(one[3], logp[1, 2])


@pytest.mark.parametrize('precision', [0, 1, 2])
def test_same_seed_same_actions_as_rsample(cuda, precision):
    O, A, B = 60, 8, 4097
    m = _model(cuda, O, A, precision)
    actor, _ = _reference(m)
    obs = torch.randn(B, O, device=cuda).clamp_(-5, 5)
    with torch.no_grad():
        mean_ref = actor.mean(obs.double()).float()
    std = torch.exp(m.named_views('actor')['log_std'])
    for s in (0, 7):
        torch.manual_seed(s)
        act, _, _, logp = m.step(obs)
        after_step = torch.cuda.get_rng_state()
        torch.manual_seed(s)
        ref = Normal(mean_ref, std).rsample()
        assert torch.equal(torch.cuda.get_rng_state(), after_step)    # the same draws from torch's generator
        _close(act, ref, 2e-5 if precision != 1 else TOL[1], f'rsample seed {s}')
        torch.manual_seed(s)
        act1 = m.actor.predict(obs)
        assert torch.equal(act1, act)
        _close(m.actor.log_prob(act1), logp, 0.0, 'log_prob of the sample')
    torch.manual_seed(3)                                              # one observation [O]: rsample draws shape [A]
    a1 = m.step(obs[0])[0]
    torch.manual_seed(3)
    _close(a1, Normal(mean_ref[0], std).rsample(), 2e-5 if precision != 1 else TOL[1], 'rsample of one row')


def _synthetic_epoch(dev, N, T, O, A, precision, eps):
    from omnisafe_b200.adapter.onpolicy_adapter import OnPolicyAdapter
    from omnisafe_b200.common.buffer import VectorOnPolicyBuffer

    cfgs = NS(algo_cfgs=NS(obs_normalize=True, reward_normalize=False, cost_normalize=False),
              logger_cfgs=NS(window_lens=100), env_cfgs=dict(obs_dim=O, act_dim=A, max_episode_steps=16))
    ad = OnPolicyAdapter('SyntheticBox-v0', N, 1, cfgs, device=dev)
    ad.precision = precision
    agent = _model(dev, O, A, precision)
    buf = VectorOnPolicyBuffer(O, A, T, 0.99, 0.95, 0.95, 'gae', 0.0, True, True, num_envs=N, device=dev)
    ad.rollout(T, agent, buf, eps=eps)
    return agent, buf


def _external_epoch(dev, N, T, O, A, precision, eps):
    from omnisafe_b200.adapter.external_adapter import ExternalEnvAdapter
    from omnisafe_b200.common.buffer import VectorOnPolicyBuffer

    cfgs = NS(algo_cfgs=NS(obs_normalize=True, reward_normalize=False, cost_normalize=False),
              logger_cfgs=NS(window_lens=100), env_cfgs=dict(obs_dim=O, act_dim=A))
    ad = ExternalEnvAdapter(xe.WIDE_BOX_ID, N, 4, cfgs, device=dev)
    ad.precision = precision
    agent = _model(dev, O, A, precision)
    buf = VectorOnPolicyBuffer(O, A, T, 0.99, 0.95, 0.95, 'gae', 0.0, True, True, num_envs=N, device=dev)
    ad.rollout(T, agent, buf, eps=eps)
    return agent, buf


@pytest.mark.parametrize('precision', [0, 1, 2])
@pytest.mark.parametrize('env', ['synthetic', 'widebox'])
def test_agrees_with_rollout(cuda, precision, env):
    N, T = 300, 8
    O, A = (60, 8) if env == 'synthetic' else (45, 3)
    eps = torch.randn(T, N, A, device=cuda)
    agent, buf = (_synthetic_epoch if env == 'synthetic' else _external_epoch)(cuda, N, T, O, A, precision, eps)
    torch.cuda.synchronize()
    d = buf.data
    bitwise = True
    for t in range(T):
        out = agent._launch(d['obs'][t].contiguous(), 7, eps=eps[t].contiguous(), act=True, logp=True)
        for k, slab in (('act', 'act'), ('logp', 'logp'), ('value_r', 'value_r'), ('value_c', 'value_c')):
            _close(out[k], d[slab][t], 2e-5, f'{env} precision {precision} t {t} {k}')
            bitwise &= torch.equal(out[k], d[slab][t])
    print(f'{env} precision {precision}: policy step vs rollout slabs bit for bit: {bitwise}')
    if precision != 0:      # the tensor-core modes run one forward (csrc/tc_forward.cuh) in both kernels
        assert bitwise


@pytest.mark.parametrize('precision,O', [(1, 60), (1, 111), (1, 376), (2, 17), (2, 60), (2, 64)])
def test_eval_snapshot_is_the_policy_mean(cuda, precision, O):
    """The evaluation kernel's old-policy snapshot (mu_store) and the policy step's mean are one function, bit for bit."""
    from omnisafe_b200._lib import lib, ptr

    A, B = 6, 1000
    m = _model(cuda, O, A, precision)
    obs = torch.randn(B, O, device=cuda).clamp_(-5, 5)
    mean = m._launch(obs, 1, mean=True)['mean']
    mu = torch.full((B, A), float('nan'), device=cuda)
    fn = lib().osb_actor_eval_x3 if precision == 2 else lib().osb_actor_eval_tc
    rc = fn(ptr(m.theta), O, A, ptr(obs), 0, 0, 0, 0, 0, 0, 0, 0, B, 1, ptr(mu), 0, 0,
            torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    torch.cuda.synchronize()
    assert torch.equal(mu, mean)


@pytest.mark.parametrize('precision', [0, 1, 2])
def test_cuda_graph_replay_gives_the_eager_bits(cuda, precision):
    from omnisafe_b200._lib import lib

    O, A, B = 60, 8, 4097
    m = _model(cuda, O, A, precision)
    lib().osb_policy_prepare()
    obs = torch.randn(B, O, device=cuda).clamp_(-5, 5)
    eps = torch.randn(B, A, device=cuda)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        m._launch(obs, 7, eps=eps, act=True, logp=True)           # warm-up on the capturing stream
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = m._launch(obs, 7, eps=eps, act=True, logp=True)
    for r in range(3):
        eps.copy_(torch.randn(B, A, device=cuda))
        g.replay()
        want = m._launch(obs, 7, eps=eps, act=True, logp=True)
        torch.cuda.synchronize()
        for k in ('act', 'logp', 'value_r', 'value_c'):
            assert torch.equal(out[k], want[k]), (r, k)
    gd = torch.cuda.CUDAGraph()                                  # deterministic step through the public method
    with torch.cuda.graph(gd):
        det = m.step(obs, deterministic=True)
    gd.replay()
    want = m.step(obs, deterministic=True)
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(det, want))


def _train_two_epochs(dev, act_between):
    """Two Philox-mode PPO-Lag epochs (rollout -> GAE -> update); `act_between` calls step(obs, True) on every slab
    row after each rollout, before the update."""
    from omnisafe_b200.algorithms.engine import UpdateEngine
    from omnisafe_b200.common.lagrange import Lagrange

    N, T, O, A = 256, 16, 60, 8
    from omnisafe_b200.adapter.onpolicy_adapter import OnPolicyAdapter
    from omnisafe_b200.common.buffer import VectorOnPolicyBuffer

    cfgs = NS(algo_cfgs=NS(obs_normalize=True, reward_normalize=False, cost_normalize=False),
              logger_cfgs=NS(window_lens=100), env_cfgs=dict(obs_dim=O, act_dim=A, max_episode_steps=16))
    ad = OnPolicyAdapter('SyntheticBox-v0', N, 1, cfgs, device=dev)
    agent = _model(dev, O, A, 2)
    buf = VectorOnPolicyBuffer(O, A, T, 0.99, 0.95, 0.95, 'gae', 0.0, True, True, num_envs=N, device=dev)
    eng = UpdateEngine(agent, buf)
    eng.precision = 2
    lag = Lagrange(25.0, 0.001, 0.035, device=dev)
    snaps = []
    for _ in range(2):
        ad.rollout(T, agent, buf)
        if act_between:
            rng = torch.cuda.get_rng_state()
            for t in range(T):
                agent.step(buf.data['obs'][t], deterministic=True)
            agent.actor.predict(buf.data['obs'].reshape(-1, O), deterministic=True)
            agent.reward_critic(buf.data['obs'][0])
            assert torch.equal(torch.cuda.get_rng_state(), rng)        # deterministic calls draw no noise
        buf.finish_paths()
        buf.finalize_statistics()
        lag.update_lagrange_multiplier(ad.window_sums)
        eng.ppo_epoch(loss_kind=0, lagrange=lag.state, net_mask=7, batch_size=1024, update_iters=2, clip=0.2,
                      critic_norm_coef=0.001, max_grad_norm=40.0, lr_actor=3e-4, lr_critic=3e-4, target_kl=0.02)
        torch.cuda.synchronize()
        snaps.append({**{k: v.clone() for k, v in buf.data.items() if v is not None},
                      'theta': agent.theta.clone(), 'adam_m': agent.adam_m.clone(), 'adam_v': agent.adam_v.clone(),
                      'norm_mean': ad._obs_normalizer.mean.clone()})
    return snaps


def test_acting_between_epochs_leaves_training_untouched(cuda):
    plain, acted = _train_two_epochs(cuda, False), _train_two_epochs(cuda, True)
    for e in range(2):
        assert plain[e].keys() == acted[e].keys()
        for k in plain[e]:
            assert torch.equal(plain[e][k], acted[e][k]), (e, k)
    assert not torch.equal(plain[0]['act'], plain[1]['act'])


def test_checkpoint_actor_acts_like_the_model(cuda, tmp_path):
    import omnisafe_b200
    from omnisafe_b200.common.normalizer import Normalizer

    N, T = 64, 32
    custom = {
        'seed': 3,
        'train_cfgs': {'device': 'cuda', 'vector_env_nums': N, 'total_steps': N * T * 2, 'parallel': 1},
        'algo_cfgs': {'steps_per_epoch': N * T, 'batch_size': 256, 'update_iters': 3},
        'logger_cfgs': {'log_dir': str(tmp_path), 'save_model_freq': 1, 'window_lens': 100, 'use_tensorboard': False},
        'env_cfgs': {'obs_dim': 45, 'act_dim': 3, 'max_episode_steps': 7},
    }
    agent = omnisafe_b200.Agent('PPOLag', xe.WIDE_BOX_ID, custom_cfgs=custom)
    agent.learn()
    model = agent.agent._actor_critic
    ckpt = torch.load(os.path.join(agent.agent.logger.log_dir, 'torch_save', 'epoch-2.pt'), weights_only=False)
    nz = Normalizer((45,), device=cuda)
    nz.load_state_dict(ckpt['obs_normalizer'])
    actor = torch.nn.Module()                               # the reference GaussianLearningActor's parameter layout
    actor.mean = torch.nn.Sequential(torch.nn.Linear(45, 64), torch.nn.Tanh(), torch.nn.Linear(64, 64), torch.nn.Tanh(),
                                     torch.nn.Linear(64, 3))
    actor.log_std = torch.nn.Parameter(torch.zeros(3))
    actor.load_state_dict(ckpt['pi'])
    actor.double().to(cuda)
    raw = torch.randn(1000, 45, device=cuda) * nz.std + nz.mean
    obs = ((raw - nz.mean) / nz.std).clamp(-5.0, 5.0)       # ObsNormalize (normalizer.py:L122-139)
    with torch.no_grad():
        want = actor.mean(obs.double())
    got = model.actor.predict(obs, deterministic=True)
    _close(got, want, TOL[model.precision], f'checkpoint actor (precision {model.precision})')
    assert model.actor.std == pytest.approx(float(torch.exp(ckpt['pi']['log_std']).mean()), rel=1e-6)
