"""GPU: the LPIPS target cache (LPIPS.cache_targets, csrc/dbw_lpips.cu dbw_lpips_forward_cached / _backward_cached).  The
cached term must equal the uncached one bit for bit -- value and d/d in1 -- whatever mix of hits and misses a batch holds;
an image one bit away from a cached one is a miss; a change of the weights drops the cache; hits skip the in0 trunk; and
the model's eager and graph-captured steps give the losses and leaf gradients of the same steps without the cache."""
import pytest
import torch

from oracle import lpips as OL

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')


@pytest.fixture(scope='module')
def sd():
    return OL.random_state_dict(0)


def _nets(sd):
    from dbw_b200.perceptual import LPIPS
    return LPIPS.from_state_dict(sd).to(DEV), LPIPS.from_state_dict(sd).to(DEV)      # cached, reference


def _imgs(n, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(n, 3, H, W, generator=g).to(DEV)


def _run(net, a, b, train, normalize, seed=1234):
    net.train(train)
    net.seed.fill_(seed)
    x = b.clone().requires_grad_(True)
    v = net(a, x, normalize=normalize)
    (v.flatten() * torch.linspace(0.5, 1.5, v.shape[0], device=DEV)).sum().backward()
    return v.detach(), x.grad


def _batches(pool, others):
    """(name, in0, expected hits): all hits in a shuffled order, all misses, hits and misses at random positions, one cached
    image repeated, and more images than the cache holds"""
    N = len(pool)
    g = torch.Generator().manual_seed(3)
    perm = torch.randperm(N, generator=g)
    mix_pick = torch.tensor([1, 0, 0, 1, 1, 0])
    mixed = torch.stack([pool[i % N] if k else others[i] for i, k in enumerate(mix_pick.tolist())])
    big = torch.cat([pool[perm], others[:2], pool[:3]])
    return [('all_hit', pool[perm], N), ('all_miss', others, 0), ('mixed', mixed, int(mix_pick.sum())),
            ('repeat', pool[2:3].expand(4, -1, -1, -1).contiguous(), 4), ('B_gt_N', big, N + 3)]


@pytest.mark.parametrize('H,W', [(40, 56), (37, 50)])             # 37x50 floors at every pool: 18x25, 9x12, 4x6, 2x3
@pytest.mark.parametrize('normalize', [True, False])
@pytest.mark.parametrize('train', [False, True])
def test_cached_term_is_the_uncached_term_bit_for_bit(sd, H, W, normalize, train):
    net, ref = _nets(sd)
    pool, others = _imgs(5, H, W, 1), _imgs(6, H, W, 2)
    net.cache_targets(pool, normalize=normalize)
    for name, a, n_hits in _batches(pool, others):
        b = (a + 0.1 * _imgs(len(a), H, W, 9 + len(a))).clamp(0, 1)
        v, g = _run(net, a, b, train, normalize)
        rv, rg = _run(ref, a, b, train, normalize)
        assert int(net.target_hits.item()) == n_hits, name
        assert torch.equal(v, rv), (name, (v - rv).abs().max().item())
        assert torch.equal(g, rg), (name, (g - rg).abs().max().item())
        assert int(net.seed.item()) == 1235
    # the other normalize, or another size: the uncached path (the hit counter is not written)
    net.target_hits.fill_(-1)
    v, g = _run(net, pool, others[:5], train, not normalize)
    rv, rg = _run(ref, pool, others[:5], train, not normalize)
    assert torch.equal(v, rv) and torch.equal(g, rg) and int(net.target_hits.item()) == -1


def test_one_bit_away_is_a_miss(sd):
    net, ref = _nets(sd)
    pool = _imgs(3, 32, 48, 4)
    net.cache_targets(pool)
    near = pool.clone()
    flat = near.view(-1).view(torch.int32)
    flat[1 * 3 * 32 * 48 + 777] ^= 1                               # image 1: one mantissa bit flipped
    b = _imgs(3, 32, 48, 5)
    v, g = _run(net, near, b, True, True)
    rv, rg = _run(ref, near, b, True, True)
    assert int(net.target_hits.item()) == 2
    assert torch.equal(v, rv) and torch.equal(g, rg)


def test_a_change_of_weights_drops_the_cache(sd):
    from dbw_b200.perceptual import LPIPS
    net, _ = _nets(sd)
    pool = _imgs(3, 32, 48, 6)
    b = _imgs(3, 32, 48, 7)
    net.cache_targets(pool)
    v_old, _ = _run(net, pool, b, False, True)
    sd1 = OL.random_state_dict(1)
    net.load_state_dict(sd1)                                      # as a reference checkpoint loaded after registration
    v, g = _run(net, pool, b, False, True)
    rv, rg = _run(LPIPS.from_state_dict(sd1).to(DEV), pool, b, False, True)
    assert torch.equal(v, rv) and torch.equal(g, rg)
    assert not torch.equal(v, v_old)
    assert net.target_hits is None                                # dropped, not served stale
    net.cache_targets(pool)
    v2, g2 = _run(net, pool, b, False, True)
    assert int(net.target_hits.item()) == 3 and torch.equal(v2, rv) and torch.equal(g2, rg)
    net.clear_target_cache()
    assert net.target_hits is None


def test_hits_skip_the_in0_trunk(sd):
    """one profiled call each: with all hits the in0 chain's bounded convolutions exit at once"""
    from torch.profiler import ProfilerActivity, profile
    net, _ = _nets(sd)
    pool, others = _imgs(4, 128, 160, 8), _imgs(4, 128, 160, 9)
    net.cache_targets(pool)
    net.eval()

    def bounded_conv_us(a):
        with torch.no_grad():
            net(a, others, normalize=True)                        # warm-up
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                net(a, others, normalize=True)
                torch.cuda.synchronize()
        ev = [e for e in prof.key_averages() if 'lpips_conv3x3_kernel' in e.key and 'true' in e.key]
        assert ev, [e.key for e in prof.key_averages()]
        return sum(e.device_time_total if hasattr(e, 'device_time_total') else e.cuda_time_total for e in ev)
    t_hit = bounded_conv_us(pool)
    assert int(net.target_hits.item()) == 4
    t_miss = bounded_conv_us(others)
    assert int(net.target_hits.item()) == 0
    print(f'in0 trunk convolutions: all hits {t_hit:.0f} us, all misses {t_miss:.0f} us')
    assert t_hit < 0.1 * t_miss


def test_cached_term_against_oracle(sd):
    """the whole-term bounds and a case of tests/test_lpips_gpu.py, the batch's first image a miss and its second a hit"""
    from tests.test_lpips_gpu import _images
    net, _ = _nets(sd)
    a, b = _images(2, 64, 96, 64 + 96)
    a, b = a.to(DEV), b.to(DEV)
    net.cache_targets(torch.cat([_imgs(1, 64, 96, 10), a[1:]]))
    gv = torch.linspace(0.5, 1.5, 2)
    net.train()
    net.seed.fill_(1234)
    x = b.clone().requires_grad_(True)
    v = net(a, x, normalize=True)
    (v.flatten() * gv.to(DEV)).sum().backward()
    assert int(net.target_hits.item()) == 1
    wv, wg = OL.value_and_grad(sd, a, b, normalize=True, mode='tf32', seed=1234, grad_value=gv)
    ev = float(((v.detach().flatten().double().cpu() - wv.cpu()).abs() / wv.cpu().abs()).max())
    eg = float((x.grad.double().cpu() - wg.cpu()).norm() / wg.cpu().norm())
    print(f'cached term: value rel {ev:.2e}, grad rel L2 {eg:.2e}')
    assert ev < 1e-4 and eg < 6e-2


# ------------------------------------------------------------------------------------------------ model steps
def _model(fine):
    from dbw_b200.dbw import PerceptualTerm
    from dbw_b200.perceptual import LPIPS
    from tests.test_model_gpu import _model_and_oracle
    model, _, _, dev = _model_and_oracle(fine=fine)
    net = LPIPS.from_state_dict(OL.random_state_dict(2))
    model.set_perceptual_loss(PerceptualTerm(net).to(dev))
    model.loss_weights = {'rgb': 1.0, 'perceptual': 0.1}
    model.train()
    return model, net


def _grads(model):
    return {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None}


def _check_same(got, want, again, what):
    """the perceptual loss bit for bit.  The other losses and the leaf gradients go through the renderer, whose backward
    accumulates with atomics: bit for bit wherever two uncached steps agree bit for bit, else within 1e-5 (relative L2) of
    the uncached step -- the run-to-run spread of those atomics"""
    (gl, gg), (wl, wg), (al, ag) = got, want, again
    assert torch.equal(gl['perceptual'], wl['perceptual']), what
    for g, w, a in ((gl, wl, al), (gg, wg, ag)):
        assert g.keys() == w.keys()
        for n in w:
            if not torch.equal(g[n], w[n]):
                print(f'{what}: {n} differs by {(g[n] - w[n]).abs().max().item():.3e} (uncached twice: '
                      f'{(a[n] - w[n]).abs().max().item():.3e})')
            assert (g[n] - w[n]).norm() <= 1e-5 * w[n].norm() + 1e-30, (what, n)


@pytest.mark.parametrize('fine', [False, True])
def test_model_step_with_a_cache_is_the_step_without(fine):
    from tests.test_model_gpu import _inputs
    model, net = _model(fine)
    inp, *_ = _inputs(model.alpha_logit.device)

    def step():
        model.zero_grad(set_to_none=True)
        net.seed.fill_(99)
        losses = model(inp, None)
        losses['total'].backward()
        return {k: v.detach().clone() for k, v in losses.items()}, _grads(model)
    want, again = step(), step()
    extra = torch.rand(2, 3, 48, 64, generator=torch.Generator().manual_seed(1)).to(inp['imgs'].device)
    nbytes = model.cache_perceptual_targets([{'imgs': x} for x in torch.cat([extra, inp['imgs'].flip(0)])])
    assert nbytes == net.target_cache_bytes(48, 64, 5)
    got = step()
    assert int(net.target_hits.item()) == len(inp['imgs'])
    _check_same(got, want, again, f'eager fine={fine}')


def test_graphed_step_with_a_cache_hits_misses_and_mixes():
    """a step captured before registration keeps computing its targets; one captured after reads the cache.  Both replay
    batches that hit, miss and mix, with the losses and gradients of the uncached step"""
    from dbw_b200.graph import GraphedStep
    from dbw_b200.parallel import ViewParallel
    from tests.test_model_gpu import _inputs
    model, net = _model(False)
    inp, *_ = _inputs(model.alpha_logit.device)
    vp = ViewParallel(model, seed=5)
    before = GraphedStep(vp, inp, len(inp['imgs']))
    pool = inp['imgs'].clone()
    model.cache_perceptual_targets(pool)
    after = GraphedStep(vp, inp, len(inp['imgs']))
    fresh = torch.rand(3, 3, 48, 64, generator=torch.Generator().manual_seed(2)).to(pool.device)
    batches = [('hit', pool.flip(0), 3), ('miss', fresh, 0), ('mix', torch.stack([fresh[0], pool[1], fresh[2]]), 1)]

    def replay(step, imgs):
        net.seed.fill_(7)
        losses = step.run(dict(inp, imgs=imgs))
        return ({k: v.detach().clone() for k, v in losses.items()},
                {str(i): g.clone() for i, g in enumerate(step.grads) if g is not None})
    for name, imgs, n_hits in batches:
        want, again = replay(before, imgs), replay(before, imgs)
        net.target_hits.fill_(-1)
        got = replay(after, imgs)
        torch.cuda.synchronize()
        assert int(net.target_hits.item()) == n_hits, name
        _check_same(got, want, again, f'graphed {name}')
