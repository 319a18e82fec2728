"""GPU parity of the scene model (DifferentiableBlocksWorld drop-in) against the oracle's restatement of
src/model/dbw.py: predict(), the RGB loss and its gradients down to the leaf parameters."""
import pytest
import torch

from oracle import dbw_path as D

pytestmark = pytest.mark.gpu

CFG = {
    'mesh': {'n_blocks': 5, 'S_world': 0.5, 'R_world': [115, 0, 0], 'txt_size': 32},
    'renderer': {'faces_per_pixel': 10, 'cameras': {'name': 'perspective'}, 'detach_bary': True, 'z_clip': 0.001},
    'rend_optim': {'coarse_learning': 1500, 'decimate_txt': 750, 'decimate_factor': 8, 'kill_blocks': True,
                   'decouple_rendering': True, 'opacity_noise': False},
    'loss': {'rgb_weight': 1, 'parsimony_weight': 0.01, 'tv_weight': 0.1, 'overlap_weight': 1},
}


def _model_and_oracle(dtype=torch.float64, fine=False, seed=5):
    import dbw_b200
    from dbw_b200.dbw import DifferentiableBlocksWorld
    from copy import deepcopy
    torch.manual_seed(seed)
    dev = torch.device('cuda:0')
    model = DifferentiableBlocksWorld((48, 64), **deepcopy(CFG)).to(dev)
    model.train()
    if fine:
        model.set_cur_epoch(2000)
        with torch.no_grad():
            model.alpha_logit.copy_(torch.tensor([2., -2., 1., 3., -1.]))
    tpl = D.SceneTemplate(n_blocks=5, txt_size=32)
    p = {k: v.detach().cpu().to(dtype).clone().requires_grad_(True) for k, v in model.named_parameters()}
    return model, tpl, p, dev


def _inputs(dev, B=3, size=(48, 64), dtype=torch.float64, seed=7):
    R, T, K = D.ring_cameras(B, dtype=dtype, jitter=0.3, seed=seed)
    g = torch.Generator().manual_seed(seed)
    imgs = torch.rand(B, 3, *size, generator=g, dtype=dtype)
    inp = {'imgs': imgs.float().to(dev), 'R': R.float().to(dev), 'T': T.float().to(dev), 'K': K.float()[None].expand(B, -1, -1).to(dev)}
    return inp, imgs, R, T, K


def test_buffers_match_oracle_template():
    model, tpl, p, dev = _model_and_oracle()
    assert torch.equal(model.sq_eta.cpu(), tpl.sq_eta) and torch.equal(model.sq_omega.cpu(), tpl.sq_omega)
    assert torch.equal(model.block_faces_uvs.cpu(), tpl.block_faces_uvs)
    assert torch.allclose(model.block_verts_uvs.cpu(), tpl.block_verts_uvs, atol=0)
    assert torch.allclose(model.R_world.cpu(), tpl.R_world, atol=1e-7)
    assert torch.equal(model.bkg_verts_uvs.cpu(), tpl.bkg_verts_uvs) and torch.equal(model.ground_verts_uvs.cpu(), tpl.ground_verts_uvs)
    assert model.txt_padding == tpl.txt_padding and model.BNF == tpl.BNF


@pytest.mark.parametrize('fine', [False, True])
def test_predict_and_rgb_gradients(fine):
    model, tpl, p, dev = _model_and_oracle(fine=fine)
    inp, imgs, R, T, K = _inputs(dev)
    decim = 8 if not fine else 0                          # decimate_txt is live below epoch 750 in training mode
    keep = None
    if fine:
        keep = torch.sigmoid(p['alpha_logit'].detach()) > 0.5
    elif CFG['rend_optim']['kill_blocks']:
        keep = torch.sigmoid(p['alpha_logit'].detach()) > 0.01
    sigma = 5e-6 if fine else 1e-4
    rec_ref = D.predict(tpl, p, R, T, K, (48, 64), sigma=sigma, faces_per_pixel=10, z_clip=0.001, fine=fine, keep=keep,
                        decimate=decim)
    rec = model.predict(inp).detach().cpu().double()
    err = (rec - rec_ref.detach()).abs()
    assert (err > 1e-4).float().mean().item() < 1e-3, f'max err {err.max().item():.3e}'
    # loss + gradients: only the rgb term (the regularisers have their own test).  The few pixels where fp32 takes a different
    # discrete decision than the fp64 oracle (colour off by > 1e-4) get a target equal to each side's own reconstruction:
    # zero residual, zero gradient on BOTH sides -- everything else must agree to the north star's 1e-3
    bad = (err > 1e-4).any(1, keepdim=True)
    print(f'decision-masked pixels: {bad.double().mean().item() * 100:.4f}%')
    inp['imgs'] = torch.where(bad, rec, imgs).float().to(dev)
    model.loss_weights = {'rgb': 1.0}
    losses = model(inp, None)
    loss_ref = D.mse_loss(torch.where(bad, rec_ref.detach(), imgs), rec_ref)
    assert abs(losses['rgb'].item() - loss_ref.item()) < 1e-5 * max(1.0, abs(loss_ref.item()))
    losses['total'].backward()
    loss_ref.backward()
    for name, prm in model.named_parameters():
        g_ref = p[name].grad
        g = prm.grad
        if g_ref is None or g_ref.abs().max() == 0:
            assert g is None or g.abs().max().item() < 1e-12, name
            continue
        rel = ((g.cpu().double() - g_ref).norm() / g_ref.norm()).item()
        assert rel < 1e-3, f'{name}: rel grad err {rel:.3e}'


def test_full_loss_dict_runs_and_is_finite():
    model, tpl, p, dev = _model_and_oracle()
    inp, *_ = _inputs(dev)
    losses = model(inp, None)
    assert set(losses) == {'rgb', 'parsimony', 'tv', 'overlap', 'total'}
    losses['total'].backward()
    for n, prm in model.named_parameters():
        assert prm.grad is not None and torch.isfinite(prm.grad).all(), n


def test_static_topology_equals_filtered_meshes():
    """blocks dropped by the opacity filters: disabling their faces (static shapes, no host sync) == removing them."""
    model, tpl, p, dev = _model_and_oracle(fine=True)
    inp, *_ = _inputs(dev)
    model.loss_weights = {'rgb': 1.0}
    outs = []
    for static in (True, False):
        model.static_topology = static
        model.zero_grad(set_to_none=True)
        losses = model(inp, None)
        losses['total'].backward()
        outs.append((losses['rgb'].item(), {n: prm.grad.clone() for n, prm in model.named_parameters() if prm.grad is not None}))
    assert abs(outs[0][0] - outs[1][0]) < 1e-7
    for n in outs[1][1]:
        a, b = outs[0][1][n], outs[1][1][n]
        assert (a - b).norm() <= 1e-4 * b.norm() + 1e-12, n


def test_cuda_graph_step_equals_eager_step():
    from dbw_b200.parallel import ViewParallel
    from dbw_b200.graph import GraphedStep
    model, tpl, p, dev = _model_and_oracle()
    inp, *_ = _inputs(dev)
    model.loss_weights = {'rgb': 1.0}
    vp = ViewParallel(model, seed=5)
    graphed = GraphedStep(vp, inp, len(inp['imgs']))
    losses = graphed.run()
    g_graph = vp.bucket.grads_flat().clone()
    noise = model.opacity_noise_buffer.clone()
    l_graph = losses['rgb'].item()
    # eager step with the same noise
    model.opacity_noise_buffer = noise
    for q in model.parameters():
        q.grad = None
    l = model(inp, None)
    l['total'].backward()
    assert abs(l['rgb'].item() - l_graph) < 1e-7
    assert (vp.bucket.grads_flat() - g_graph).norm() <= 1e-4 * g_graph.norm()
    # replay with new inputs changes the result, and is repeatable
    inp2 = {k: (v.flip(0).contiguous() if k in ('imgs',) else v) for k, v in inp.items()}
    l2 = graphed.run(inp2)['rgb'].item()
    assert abs(l2 - l_graph) > 1e-9


def test_fused_scene_geometry_matches_torch_path():
    """dbw_scene_geometry_* (one kernel each way) with an empty static environment vs the eager restatement of
    dbw.py:299-311,344,348-352; with the background sphere's vertices ahead of the ground, the ground, the blocks and the
    leaf gradients are the same bits"""
    from dbw_b200 import geometry as G
    from dbw_b200.scene_ops import scene_geometry_passes
    model, tpl, p, dev = _model_and_oracle()
    with torch.no_grad():
        model.sq_eps.copy_(torch.randn_like(model.sq_eps))
        model.R_6d_ground.add_(0.1 * torch.randn_like(model.R_6d_ground))
    st = model._fused_arrays()
    leaves = [model.sq_eps, model.S, model.R_6d, model.T, model.R_6d_ground, model.T_ground]
    blk, ground = scene_geometry_passes(*leaves, st['geom'], torch.zeros(0, 3, device=dev))
    out = torch.cat([blk, ground])
    # eager
    S, R, T = model.S.exp() + model.scale_min, G.rotation_6d_to_matrix(model.R_6d), model.T
    vb = model._to_world((model.get_blocks_verts() * S[:, None]) @ R + T[:, None]).reshape(-1, 3)
    gv = model.ground.get_mesh_verts_faces(0)[0][None]
    vg = model._to_world(gv @ G.rotation_6d_to_matrix(model.R_6d_ground) + model.T_ground[:, None])[0]
    ref = torch.cat([vb, vg])
    assert (out - ref).abs().max().item() < 2e-6
    w = torch.randn_like(ref)
    g_f = torch.autograd.grad((out * w).sum(), leaves)
    g_r = torch.autograd.grad((ref * w).sum(), leaves)
    for a, b, n in zip(g_f, g_r, ['sq_eps', 'S', 'R_6d', 'T', 'R_6d_ground', 'T_ground']):
        assert (a - b).norm() <= 2e-5 * b.norm() + 1e-7, (n, (a - b).norm().item(), b.norm().item())
    bkg = st['bkg_world']
    blk_s, env_s = scene_geometry_passes(*leaves, st['geom'], bkg)
    assert torch.equal(blk_s, blk) and torch.equal(env_s, torch.cat([bkg, ground]))
    w_env = torch.cat([torch.randn_like(bkg), w[blk.shape[0]:]])
    g_s = torch.autograd.grad((blk_s * w[:blk.shape[0]]).sum() + (env_s * w_env).sum(), leaves)
    for a, b in zip(g_s, g_f):
        assert torch.equal(a, b)


@pytest.mark.parametrize('decim', [1, 8])
@pytest.mark.parametrize('pad', [(0, 0), (0, 5), (3, 2)])
def test_fused_texture_atlas_matches_torch_path(decim, pad):
    """scene_atlases (background, ground and blocks in one launch each way) vs the eager restatement of dbw.py:331-341: the
    environment maps decimated by `decim`, the blocks' maps by 1 and by 8 and padded by `pad`"""
    import torch.nn.functional as F
    from dbw_b200.scene_ops import scene_atlases
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(3)

    def eager(tex, f, pad):
        maps = torch.sigmoid(tex)
        if f > 1:
            sub = F.avg_pool2d(maps.permute(0, 3, 1, 2), kernel_size=f, stride=f)
            maps = F.interpolate(sub, scale_factor=f).permute(0, 2, 3, 1)
        return F.pad(maps.permute(0, 3, 1, 2), pad=(pad[0], pad[1], 0, 0), mode='circular').permute(0, 2, 3, 1)

    tb, tg = (torch.randn(1, 64, 64, 3, generator=g).to(dev).requires_grad_(True) for _ in range(2))
    tk = torch.randn(3, 32, 32, 3, generator=g).to(dev).requires_grad_(True)
    for decim_blocks in (1, 8):
        env, blk = scene_atlases(tb, tg, tk, pad, decim, decim_blocks)
        ref_env, ref_blk = torch.cat([eager(tb, decim, (0, 0)), eager(tg, decim, (0, 0))]), eager(tk, decim_blocks, pad)
        assert env.shape == (2, 64, 64, 4) and blk.shape == (3, 32, 32 + sum(pad), 4)
        for atlas, ref in ((env, ref_env), (blk, ref_blk)):
            assert (atlas[..., :3] - ref).abs().max().item() < 1e-6 and (atlas[..., 3] == 0).all()
        we, wb = torch.randn(env.shape, generator=g).to(dev), torch.randn(blk.shape, generator=g).to(dev)
        ga = torch.autograd.grad((env * we).sum() + (blk * wb).sum(), [tb, tg, tk])
        gr = torch.autograd.grad((ref_env * we[..., :3]).sum() + (ref_blk * wb[..., :3]).sum(), [tb, tg, tk])
        for a, b in zip(ga, gr):
            assert (a - b).norm() <= 1e-5 * b.norm()


@pytest.mark.parametrize('fine', [False, True])
def test_fused_scene_path_equals_eager_path(fine):
    model, tpl, p, dev = _model_and_oracle(fine=fine)
    inp, *_ = _inputs(dev)
    outs = []
    for fused in (True, False):
        model.fused_scene = fused
        model.zero_grad(set_to_none=True)
        losses = model(inp, None)
        losses['total'].backward()
        outs.append(({k: v.item() for k, v in losses.items()},
                     {n: (prm.grad.clone() if prm.grad is not None else torch.zeros_like(prm)) for n, prm in model.named_parameters()}))
    for k in outs[1][0]:
        assert abs(outs[0][0][k] - outs[1][0][k]) <= 1e-6 * max(1.0, abs(outs[1][0][k])), k
    for n in outs[1][1]:
        a, b = outs[0][1][n], outs[1][1][n]
        assert (a - b).norm() <= 2e-4 * b.norm() + 1e-10, (n, (a - b).norm().item(), b.norm().item())


@pytest.mark.parametrize('fine', [False, True])
def test_loss_epilogue_in_the_rasterizer_equals_composite_kernel(fine):
    """fused_loss.scene_mse (compositing + MSE + their gradients in the blocks pass' epilogue, dbw_render_forward_loss /
    dbw_render_backward) against the separate render -> dbw_composite_mse path, incl. a non-unit upstream gradient
    and the global-batch normalisation of a view shard."""
    model, tpl, p, dev = _model_and_oracle(fine=fine)
    inp, *_ = _inputs(dev)
    model.loss_weights = {'rgb': 1.0}
    model.n_total_views = 7                      # this batch is a 3-view shard of a 7-view step
    outs = []
    for fused in (True, False):
        model.fused_loss = fused
        assert model._fused_loss_ok(inp['imgs']) == fused
        model.zero_grad(set_to_none=True)
        losses = model(inp, None)
        (0.37 * losses['total']).backward()
        outs.append((losses['rgb'].item(), {n: prm.grad.clone() for n, prm in model.named_parameters() if prm.grad is not None}))
    assert abs(outs[0][0] - outs[1][0]) <= 1e-6 * abs(outs[1][0])
    assert set(outs[0][1]) == set(outs[1][1])
    for n in outs[1][1]:
        a, b = outs[0][1][n], outs[1][1][n]
        assert (a - b).norm() <= 1e-4 * b.norm() + 1e-12, (n, (a - b).norm().item(), b.norm().item())


def test_loss_epilogue_returns_the_composited_image():
    from dbw_b200.fused_loss import scene_mse
    model, tpl, p, dev = _model_and_oracle()
    inp, *_ = _inputs(dev)
    model.eval()
    with torch.no_grad():
        rec_ref = model.predict(inp)
        model._install_cameras(inp)
        model._scene_mse_fused(inp)             # builds the pass descriptions
        _, hard_filter, _ = model._phase()
        (ev, ea, _), (bv, ba, _, fmap, alpha) = model._scene_tensors(hard_filter)
        loss, rec = scene_mse(ev, ea, bv, ba, alpha, inp['R'], inp['T'], inp['imgs'], model._passes[1], model._passes[2], fmap,
                              return_rec=True)
    assert torch.allclose(rec, rec_ref, atol=1e-6)
    assert abs(loss.item() - ((rec_ref - inp['imgs']) ** 2).mean().item()) < 1e-6


def test_composite_mse_fused_matches_torch():
    """dbw_composite_mse / _backward vs the eager expressions of dbw.py:223,366-367, incl. a gradient arriving at rec."""
    from dbw_b200.dbw import _CompositeMSE
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(0)
    fg = torch.rand(3, 4, 20, 28, generator=g).to(dev).requires_grad_(True)
    env = torch.rand(3, 4, 20, 28, generator=g).to(dev).requires_grad_(True)
    imgs = torch.rand(3, 3, 20, 28, generator=g).to(dev)
    w = torch.rand(3, 3, 20, 28, generator=g).to(dev)
    rec, loss = _CompositeMSE.apply(fg, env, imgs, 5)
    (0.7 * loss + (rec * w).sum()).backward()
    a = (fg.grad.clone(), env.grad.clone()); fg.grad = None; env.grad = None
    rec_t = fg[:, :3] * fg[:, 3:] + (1 - fg[:, 3:]) * env[:, :3]
    loss_t = ((imgs - rec_t) ** 2).sum() / (5 * 3 * 20 * 28)
    (0.7 * loss_t + (rec_t * w).sum()).backward()
    assert torch.allclose(rec, rec_t, atol=1e-6) and abs(loss.item() - loss_t.item()) < 1e-6
    assert torch.allclose(a[0], fg.grad, atol=1e-6, rtol=1e-5) and torch.allclose(a[1], env.grad, atol=1e-6, rtol=1e-5)


def test_graphed_step_recaptures_when_the_schedule_switches_phase():
    from dbw_b200.parallel import ViewParallel
    from dbw_b200.graph import GraphedStep
    model, tpl, p, dev = _model_and_oracle()
    inp, *_ = _inputs(dev)
    model.loss_weights = {'rgb': 1.0}
    vp = ViewParallel(model, seed=5)
    graphed = GraphedStep(vp, inp, len(inp['imgs']))
    l_coarse = graphed.run()['rgb'].item()
    model.set_cur_epoch(2000)                      # past coarse_learning (1500) and decimate_txt (750)
    l_fine = graphed.run()['rgb'].item()
    model.opacity_noise_buffer = None
    ref = model(inp, None)['rgb'].item()
    assert abs(l_fine - ref) < 1e-7 and abs(l_fine - l_coarse) > 1e-9


def test_visualisation_paths_of_the_trainer_run():
    """what src/trainer.py:177-199 calls every val_stat_interval: predict(w_edges=True), predict_synthetic,
    get_arranged_block_txt -- shapes, ranges, and that the overlay only touches pixels near face edges."""
    model, tpl, p, dev = _model_and_oracle()
    inp, *_ = _inputs(dev)
    model.eval()
    with torch.no_grad():
        rec = model.predict(inp, None)
        rec_e = model.predict(inp, None, w_edges=True)
        syn = model.predict_synthetic(inp, None)
        txt = model.get_arranged_block_txt()
    assert rec.shape == rec_e.shape == syn.shape == inp['imgs'].shape and txt.shape[:2] == (1, 3)
    for t in (rec, rec_e, syn):
        assert torch.isfinite(t).all() and t.min() >= -1e-5 and t.max() <= 1 + 1e-5
    changed = ((rec - rec_e).abs().max(1)[0] > 1e-6).float().mean().item()
    assert 0.005 < changed < 0.6                                  # lines, not areas
    white = (syn.min(1)[0] > 0.999).float().mean().item()         # white background where no opaque block is
    assert 0.1 < white < 0.99
    cols = model.get_scene_face_colors()
    assert cols.shape == (model.env_n_faces + model.blocks_n_faces, 3) and cols.min() >= 0 and cols.max() <= 1


def test_optimisation_descends_with_the_reference_optimizer_layout():
    """a short optimisation exactly as src/trainer.py:137-147 + src/optimizer.py:9-14 drive it (Adam, texture group with its
    own lr): targets rendered from a perturbed copy of the scene; the loss must keep descending."""
    from copy import deepcopy
    from dbw_b200.dbw import DifferentiableBlocksWorld
    dev = torch.device('cuda:0')
    cfg = deepcopy(CFG)
    cfg['rend_optim']['opacity_noise'] = False
    torch.manual_seed(1)
    target_model = DifferentiableBlocksWorld((48, 64), **deepcopy(cfg)).to(dev)
    target_model.eval()
    inp, *_ = _inputs(dev, B=4)
    with torch.no_grad():
        inp['imgs'] = target_model.predict(inp, None).clamp(0, 1)
    torch.manual_seed(2)
    model = DifferentiableBlocksWorld((48, 64), **deepcopy(cfg)).to(dev)
    model.train()
    named = list(model.named_parameters())
    opt = torch.optim.Adam([dict(params=[p for n, p in named if not n.startswith('texture')]),
                            dict(params=[p for n, p in named if n.startswith('texture')], lr=5e-2)], lr=5e-3)
    hist = []
    for it in range(60):
        opt.zero_grad()
        loss = model(inp, None)
        loss['total'].backward()
        opt.step()
        hist.append(loss['rgb'].item())
    assert all(torch.isfinite(p).all() for p in model.parameters())
    assert hist[-1] < 0.85 * hist[0] and min(hist[-10:]) < min(hist[:10]), (hist[0], hist[-1])   # measured: 1.01e-3 -> 7.4e-4


# ------------------------------------------------------------------------------------------------ branches round 1 left untested
def test_joint_render_mode_matches_oracle():
    """decouple_rendering=False (dbw.py:225-232): background + ground + blocks rendered as ONE scene by the block renderer,
    environment faces at opacity 1 -- predict() and the RGB-loss gradients against the oracle's restatement"""
    from copy import deepcopy
    from dbw_b200.dbw import DifferentiableBlocksWorld
    cfg = deepcopy(CFG)
    cfg['rend_optim'].update(decouple_rendering=False, kill_blocks=False)
    cfg['loss'] = {'rgb_weight': 1}
    torch.manual_seed(5)
    dev = torch.device('cuda:0')
    model = DifferentiableBlocksWorld((48, 64), **cfg).to(dev)
    model.train()
    tpl = D.SceneTemplate(n_blocks=5, txt_size=32)
    p = {k: v.detach().cpu().double().clone().requires_grad_(True) for k, v in model.named_parameters()}
    inp, imgs, R, T, K = _inputs(dev)
    rec_ref = D.predict_joint(tpl, p, R, T, K, (48, 64), sigma=1e-4, faces_per_pixel=10, z_clip=0.001, decimate=8)
    rec = model.predict(inp)
    err = (rec.detach().cpu().double() - rec_ref.detach()).abs()
    bad = (err > 1e-4).any(1, keepdim=True)
    assert bad.double().mean().item() < 2e-3, f'max err {err.max().item():.3e}'
    # gradients, with the (few) deviating pixels given zero residual on both sides
    inp['imgs'] = torch.where(bad, rec.detach().cpu().double(), imgs).float().to(dev)
    losses = model(inp, None)
    loss_ref = D.mse_loss(torch.where(bad, rec_ref.detach(), imgs), rec_ref)
    assert abs(losses['rgb'].item() - loss_ref.item()) < 1e-5 * max(1.0, abs(loss_ref.item()))
    losses['total'].backward()
    loss_ref.backward()
    for name, prm in model.named_parameters():
        g_ref = p[name].grad
        if g_ref is None or g_ref.abs().max() == 0:
            continue
        rel = ((prm.grad.cpu().double() - g_ref).norm() / g_ref.norm()).item()
        assert rel < 2e-3, f'{name}: rel grad err {rel:.3e}'


def test_regularisers_match_oracle_restatement():
    """parsimony / TV / overlap (dbw.py:373-405) of model(inp) against oracle.regularisers -- itself pinned to the reference's
    compute_losses in tests/test_oracle_golden.py -- values and leaf gradients, with shared overlap sample points"""
    for tv_type in ('l2sq', 'l2'):
        from copy import deepcopy
        from dbw_b200.dbw import DifferentiableBlocksWorld
        cfg = deepcopy(CFG)
        cfg['loss'] = {'rgb_weight': 1, 'parsimony_weight': 0.01, 'tv_weight': 0.1, 'overlap_weight': 1, 'tv_type': tv_type}
        torch.manual_seed(5)
        dev = torch.device('cuda:0')
        model = DifferentiableBlocksWorld((48, 64), **cfg).to(dev)
        model.train()
        with torch.no_grad():
            model.T.mul_(0.05)
            model.alpha_logit.copy_(torch.tensor([3.0, 2.5, 2.0, 1.0, -6.0]))
        tpl = D.SceneTemplate(n_blocks=5, txt_size=32)
        p = {k: v.detach().cpu().double().clone().requires_grad_(True) for k, v in model.named_parameters()}
        inp, *_ = _inputs(dev)
        u01 = torch.rand(5, 1000, 3, generator=torch.Generator().manual_seed(9))
        model.overlap_samples_buffer = u01.to(dev)
        losses = model(inp, None)
        ref = D.regularisers(tpl, p, coarse=True, keep=torch.sigmoid(p['alpha_logit'].detach()) > 0.01, tv_type=tv_type,
                             unit_samples=u01.double(), weights=(0.01, 0.1, 1.0))
        assert ref['overlap'].item() > 0
        for k in ('parsimony', 'tv', 'overlap'):
            assert abs(losses[k].item() - ref[k].item()) <= 2e-5 * max(abs(ref[k].item()), 1e-3), (tv_type, k, losses[k].item(), ref[k].item())
        (losses['parsimony'] + losses['tv'] + losses['overlap']).backward()
        sum(ref.values()).backward()
        for name, prm in model.named_parameters():
            g_ref = p[name].grad
            if g_ref is None or g_ref.abs().max() == 0:
                continue
            rel = ((prm.grad.cpu().double() - g_ref).norm() / g_ref.norm()).item()
            assert rel < 1e-3, f'{tv_type} {name}: rel grad err {rel:.3e}'


def test_perceptual_hand_off_reaches_the_leaves():
    """a stand-in perceptual callable through model(inp): `rec` feeds it, its gradient on rec enters dbw_composite_mse_backward
    (g_rec) next to the MSE's and reaches every leaf -- checked against the oracle with the same callable (dbw.py:369-371)"""
    model, tpl, p, dev = _model_and_oracle()
    inp, imgs, R, T, K = _inputs(dev)
    model.loss_weights = {'rgb': 1.0, 'perceptual': 0.1}
    g = torch.Generator().manual_seed(3)
    kern = torch.randn(4, 3, 5, 5, generator=g, dtype=torch.float64) * 0.2

    def perceptual(a, b):                      # a small fixed conv "feature" distance: smooth, touches every pixel
        k = kern.to(a)
        return (torch.nn.functional.conv2d(a, k) - torch.nn.functional.conv2d(b, k)).pow(2).mean()

    model.set_perceptual_loss(perceptual)
    assert not model._fused_loss_ok(inp['imgs'])                 # another consumer of rec: the separate composite kernel is used
    keep = torch.sigmoid(p['alpha_logit'].detach()) > 0.01
    rec_ref = D.predict(tpl, p, R, T, K, (48, 64), sigma=1e-4, faces_per_pixel=10, z_clip=0.001, keep=keep, decimate=8)
    rec = model.predict(inp).detach().cpu().double()
    bad = ((rec - rec_ref.detach()).abs() > 1e-4).any(1, keepdim=True)
    assert bad.double().mean().item() < 2e-3
    inp['imgs'] = torch.where(bad, rec, imgs).float().to(dev)
    imgs_ref = torch.where(bad, rec_ref.detach(), imgs)
    losses = model(inp, None)
    ref_p = 0.1 * perceptual(imgs_ref, rec_ref)
    ref_total = D.mse_loss(imgs_ref, rec_ref) + ref_p
    assert abs(losses['perceptual'].item() - ref_p.item()) < 2e-4 * max(abs(ref_p.item()), 1e-6)
    losses['total'].backward()
    ref_total.backward()
    for name, prm in model.named_parameters():
        g_ref = p[name].grad
        if g_ref is None or g_ref.abs().max() == 0:
            continue
        rel = ((prm.grad.cpu().double() - g_ref).norm() / g_ref.norm()).item()
        assert rel < 2e-2, f'{name}: rel grad err {rel:.3e}'      # masked pixels still carry the (dense) perceptual gradient
    # the term really contributes: dropping it changes the texture gradient
    g_with = model.textures.grad.clone()
    model.zero_grad(set_to_none=True)
    model.loss_weights = {'rgb': 1.0}
    model(inp, None)['total'].backward()
    assert (g_with - model.textures.grad).norm() > 1e-3 * g_with.norm()


def test_pipelined_steps_each_draw_their_own_opacity_noise():
    """two GraphedSteps on one model (PipelinedGraphedStep): each replays against ITS captured noise buffer, refreshed before
    every replay from a shared generator -- round 1's second capture orphaned the first one's buffer (ADVICE)"""
    from dbw_b200.parallel import ViewParallel
    from dbw_b200.graph import PipelinedGraphedStep
    model, tpl, p, dev = _model_and_oracle()
    model.opacity_noise = True
    inp, *_ = _inputs(dev)
    model.loss_weights = {'rgb': 1.0}
    vp = ViewParallel(model, seed=5)
    piped = PipelinedGraphedStep(vp, inp, len(inp['imgs']))
    host = {k: v.cpu().pin_memory() for k, v in inp.items()}
    seen = []
    for it in range(4):
        losses = piped.run(host, host)
        torch.cuda.synchronize()
        step = piped.steps[it % 2]
        assert step.noise_buf.abs().max().item() > 0                        # drawn, not the stale zeros
        assert model.opacity_noise_buffer is step.noise_buf
        seen.append((step.noise_buf.clone(), losses['rgb'].item()))
    assert all(not torch.equal(seen[i][0], seen[j][0]) for i in range(4) for j in range(i))      # consecutive draws of one generator
    assert len({round(l, 9) for _, l in seen}) == 4                         # and the loss follows the noise
    # an eager step with step 3's noise reproduces step 3's loss
    model.opacity_noise_buffer = seen[3][0]
    assert abs(model(inp, None)['rgb'].item() - seen[3][1]) < 1e-7


def test_pipelined_steps_leave_their_own_gradients_in_the_grad_attributes():
    """two GraphedSteps on one model, gradients not gathered into the bucket (one rank): after a replay the .grad attributes are
    the tensors THAT step's graph wrote -- not the other step's, which the later capture had left there"""
    from dbw_b200.parallel import ViewParallel
    from dbw_b200.graph import PipelinedGraphedStep
    model, tpl, p, dev = _model_and_oracle()
    inp, *_ = _inputs(dev)
    model.loss_weights = {'rgb': 1.0}
    vp = ViewParallel(model, seed=5)
    piped = PipelinedGraphedStep(vp, inp, len(inp['imgs']))
    host_a = {k: v.cpu().pin_memory() for k, v in inp.items()}
    host_b = dict(host_a, imgs=host_a['imgs'].flip(0).contiguous().pin_memory())
    got = []
    for cur, nxt in ((host_a, host_b), (host_b, host_a), (host_a, host_b), (host_b, None)):
        piped.run(cur, nxt)
        torch.cuda.synchronize()
        got.append(vp.bucket.grads_flat().clone())
    refs = []
    for host in (host_a, host_b):
        for q in model.parameters():
            q.grad = None
        model({k: v.to(dev) for k, v in host.items()}, None)['total'].backward()
        refs.append(vp.bucket.grads_flat().clone())
    assert (refs[0] - refs[1]).norm() > 1e-2 * refs[0].norm()
    for i, g in enumerate(got):
        ref = refs[i % 2]
        assert (g - ref).norm() <= 1e-4 * ref.norm(), (i, (g - ref).norm().item(), ref.norm().item())


def test_row_band_shards_sum_to_the_batch():
    """(view, row band) sharding (parallel.shard_row_bands + dbw_render.h view_rows): the loss and every leaf gradient of the
    full batch == the sum over 3 'ranks' that each render their bands of the views they touch"""
    from dbw_b200.parallel import shard_row_bands
    model, tpl, p, dev = _model_and_oracle()
    inp, *_ = _inputs(dev, B=3)
    model.loss_weights = {'rgb': 1.0}
    model.n_total_views = 3
    model.zero_grad(set_to_none=True)
    full = model(inp, None)
    full['total'].backward()
    g_full = {n: prm.grad.clone() for n, prm in model.named_parameters() if prm.grad is not None}
    tot, g_sum = 0.0, None
    for rank in range(3):
        pieces = shard_row_bands(3, 48, 3, rank)                # 48 rows = 3 bands per view: ranks own whole views here...
        pieces = [(v, a, b) for v, a, b in pieces]
        if rank == 0:                                            # ...so cut unevenly by hand: rank 0 gets view 0 + top of view 1
            pieces = [(0, 0, 48), (1, 0, 16)]
        elif rank == 1:
            pieces = [(1, 16, 48), (2, 0, 32)]
        else:
            pieces = [(2, 32, 48)]
        idx = [v for v, _, _ in pieces]
        local = {k: v[idx[0]:idx[-1] + 1].contiguous() for k, v in inp.items()}
        local['rows'] = torch.tensor([[a, b] for _, a, b in pieces], dtype=torch.int32, device=dev)
        model.zero_grad(set_to_none=True)
        out = model(local, None)
        out['total'].backward()
        tot += out['rgb'].item()
        g = {n: prm.grad.clone() for n, prm in model.named_parameters() if prm.grad is not None}
        g_sum = g if g_sum is None else {n: g_sum[n] + g[n] for n in g}
    assert abs(tot - full['rgb'].item()) < 1e-6 * max(1.0, abs(tot))
    for n in g_full:
        assert (g_sum[n] - g_full[n]).norm() <= 1e-4 * g_full[n].norm() + 1e-12, (n, (g_sum[n] - g_full[n]).norm().item(), g_full[n].norm().item())


def test_quantitative_and_qualitative_eval(tmp_path):
    """the two evaluation entry points the trainer calls at the end of a run (trainer.py:246-249): the final_scores.tsv columns
    of dbw.py:464-493 and the still images / OBJ meshes of dbw.py:495-554"""
    model, tpl, p, dev = _model_and_oracle(fine=True)
    inp, *_ = _inputs(dev, B=4)
    loader = [({k: v[:2].cpu() for k, v in inp.items()}, {}), ({k: v[2:].cpu() for k, v in inp.items()}, {})]
    scores = model.quantitative_eval(loader, dev, hard_inference=True)
    assert list(scores)[:6] == ['n_blocks', 'L_tot', 'L_rec', 'PSNR', 'SSIM', 'LPIPS'] and list(scores)[6:] == [f'alpha{k}' for k in range(5)]
    assert scores['n_blocks'] == 3 and 3 < scores['PSNR'] < 20 and -0.2 < scores['SSIM'] < 0.5 and scores['L_rec'] > 0
    n = model.qualitative_eval(loader, dev, path=tmp_path)
    assert n == 4
    names = {f.name for f in tmp_path.iterdir()} | {f'textures/{f.name}' for f in (tmp_path / 'textures').iterdir()}
    assert {'mesh.obj', 'mesh_full.obj', '0_inp.png', '0_rec.png', '0_rec_col.png', '0_rec_col_inp.png', '0_rec_syn_nobkg.png',
            '0_rec_syn_nobkg_edged.png', '3_rec.png', 'textures/bkg.png', 'textures/ground.png', 'textures/block_04.png'} <= names
    faces = sum(1 for l in open(tmp_path / 'mesh.obj') if l.startswith('f '))
    assert faces == 128 + 3 * 80                                   # reduced ground + the three opaque blocks


@pytest.mark.parametrize('decim', [(1, 1), (8, 8), (8, 1)])
def test_scene_atlases_one_launch_equals_three(decim):
    """dbw_texture_prep_*_multi: background + ground + blocks in one launch each way (scene_atlases) == one launch per
    stack, values and gradients bit for bit"""
    from dbw_b200._lib import DbwTexJob
    from dbw_b200.scene_ops import scene_atlases, _tex_launch
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(4)
    tb, tg = (torch.randn(1, 64, 64, 3, generator=g).to(dev).requires_grad_(True) for _ in range(2))
    tk = torch.randn(3, 32, 32, 3, generator=g).to(dev).requires_grad_(True)
    env, blk = scene_atlases(tb, tg, tk, (3, 5), decim[0], decim[1])
    we, wb = torch.randn_like(env), torch.randn_like(blk)
    ga = torch.autograd.grad((env * we).sum() + (blk * wb).sum(), [tb, tg, tk])
    ref_env, ref_blk = torch.empty_like(env), torch.empty_like(blk)
    gr = [torch.empty_like(t) for t in (tb, tg, tk)]
    stacks = ((tb, ref_env[0], we[0], 0, 0, decim[0]), (tg, ref_env[1], we[1], 0, 0, decim[0]), (tk, ref_blk, wb, 3, 5, decim[1]))
    for (t, out, w, pl, pr, f), gt in zip(stacks, gr):
        t = t.detach()
        _tex_launch([DbwTexJob(t.data_ptr(), out.data_ptr(), None, t.shape[0], t.shape[1], pl, pr, f, 0)], False)
        _tex_launch([DbwTexJob(t.data_ptr(), w.data_ptr(), gt.data_ptr(), t.shape[0], t.shape[1], pl, pr, f, 0)], True)
    assert torch.equal(env, ref_env) and torch.equal(blk, ref_blk)
    for a, b in zip(ga, gr):
        assert torch.equal(a, b)


@pytest.mark.parametrize('thr', [-1.0, 0.01, 0.5])
@pytest.mark.parametrize('noisy', [False, True])
def test_block_opacities_kernel_matches_the_eager_ops(thr, noisy):
    """dbw_opacity_forward / _backward vs the eager ops of src/model/dbw.py:300-316 (static shapes)"""
    from dbw_b200.scene_ops import block_opacities
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(11)
    N, BNF = 7, 12
    logit = (3 * torch.randn(N, generator=g)).to(dev).requires_grad_(True)
    with torch.no_grad():
        logit[2] = -6.0                                          # sigmoid = 0.0025: killed at 0.01
    noise = torch.randn(N, generator=g).to(dev) if noisy else None
    fmap0 = torch.arange(N, device=dev, dtype=torch.int32).repeat_interleave(BNF)
    alpha, kept, fmap = block_opacities(logit, noise, 0.7 if noisy else 0.0, thr, fmap0, BNF)
    ref_alpha = torch.sigmoid(logit + 0.7 * noise) if noisy else torch.sigmoid(logit)
    keep = torch.sigmoid(logit.detach()) > thr if thr >= 0 else torch.ones(N, dtype=torch.bool, device=dev)
    ref_kept = ref_alpha * keep
    ref_fmap = torch.where(keep[:, None], fmap0.view(N, BNF), torch.full((), -1, dtype=torch.int32, device=dev)).reshape(-1)
    assert (alpha - ref_alpha).abs().max().item() < 2e-7 and (kept - ref_kept).abs().max().item() < 2e-7
    assert torch.equal(fmap, ref_fmap) and (thr >= 0 or fmap.data_ptr() == fmap0.data_ptr())
    assert thr < 0.01 or not bool(keep[2])
    wa, wk = torch.randn(N, generator=g).to(dev), torch.randn(N, generator=g).to(dev)
    ga, = torch.autograd.grad((alpha * wa).sum() + (kept * wk).sum(), logit, retain_graph=True)
    gr, = torch.autograd.grad((ref_alpha * wa).sum() + (ref_kept * wk).sum(), logit, retain_graph=True)
    assert (ga - gr).abs().max().item() < 1e-6
    g_only_alpha, = torch.autograd.grad((alpha * wa).sum(), logit)          # alpha_kept unused: its gradient arrives as None
    assert (g_only_alpha - torch.autograd.grad((ref_alpha * wa).sum(), logit)[0]).abs().max().item() < 1e-6


@pytest.mark.parametrize('decim', [(1, 1), (8, 8), (8, 1)])
def test_texture_cells_then_expand_equals_the_fused_preparation(decim):
    """DBW_TEX_STAGE_CELLS + DBW_TEX_STAGE_EXPAND (the split a data-parallel step sums gradients at) == DBW_TEX_STAGE_FUSED,
    bit for bit, forward and backward"""
    from dbw_b200.scene_ops import scene_atlases, scene_texture_cells, atlases_from_cells
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(4)
    tb, tg = (torch.randn(1, 64, 64, 3, generator=g).to(dev).requires_grad_(True) for _ in range(2))
    tk = torch.randn(3, 32, 32, 3, generator=g).to(dev).requires_grad_(True)
    ref_env, ref_blk = scene_atlases(tb, tg, tk, (3, 5), decim[0], decim[1])
    cells_env, cells_blk = scene_texture_cells(tb, tg, tk, decim[0], decim[1])
    assert cells_env.shape == (2, 64 // decim[0], 64 // decim[0], 3) and cells_blk.shape == (3, 32 // decim[1], 32 // decim[1], 3)
    env, blk = atlases_from_cells(cells_env, cells_blk, (3, 5), decim[0], decim[1])
    assert torch.equal(env, ref_env) and torch.equal(blk, ref_blk)
    if decim[1] == 8:                                                      # a cell = the mean of its 8 x 8 sigmoids
        want = torch.sigmoid(tk.detach()).view(3, 4, 8, 4, 8, 3).mean(dim=(2, 4))
        assert (cells_blk - want).abs().max().item() < 1e-6
    we, wb = torch.randn_like(env), torch.randn_like(blk)
    ga = torch.autograd.grad((env * we).sum() + (blk * wb).sum(), [tb, tg, tk])
    gr = torch.autograd.grad((ref_env * we).sum() + (ref_blk * wb).sum(), [tb, tg, tk])
    for a, b in zip(ga, gr):
        assert torch.equal(a, b)


def test_gradient_sum_point_is_the_identity_on_one_rank():
    """parallel.GradSumPoint wired through the model (vertices, opacities and texture CELLS of a step go through it) with a
    one-rank stand-in for the peer-memory bucket: the step's loss equals the plain step's bit for bit, its leaf gradients to the
    rounding of the raster backward's atomics (two executions of the SAME step differ by as much), and every gradient the
    raster passes produce went through the bucket in one piece"""
    from dbw_b200.parallel import GradSumPoint
    model, tpl, p, dev = _model_and_oracle()
    inp, *_ = _inputs(dev)
    model.loss_weights = {'rgb': 1}

    class OneRankBucket:
        def __init__(self):
            self.flat = torch.zeros(model.grad_sum_floats() + 3, device=dev)
            self.calls = []

        def all_reduce(self, buf):
            assert buf.data_ptr() == self.flat.data_ptr() and buf.numel() % 4 == 0
            self.calls.append(buf.numel())

    assert model.can_sum_gradients_at_scene_tensors(inp['imgs'])
    params = [q for q in model.parameters() if q.requires_grad]
    ref_loss = model(inp)['total']
    ref = torch.autograd.grad(ref_loss, params, allow_unused=True)
    bucket = OneRankBucket()
    model.grad_sum_point = GradSumPoint(bucket)
    try:
        loss = model(inp)['total']
        got = torch.autograd.grad(loss, params, allow_unused=True)
    finally:
        model.grad_sum_point = None
    assert torch.equal(loss, ref_loss)
    assert len(bucket.calls) == 1 and bucket.calls[0] <= model.grad_sum_floats() + 3
    again = torch.autograd.grad(model(inp)['total'], params, allow_unused=True)
    for a, b, c in zip(got, ref, again):
        assert (a is None) == (b is None)
        if a is not None:
            assert (a - b).norm() <= 1e-5 * b.norm() + 4 * (c - b).norm() + 1e-12, ((a - b).norm().item(), (c - b).norm().item())
    model.set_cur_epoch(2000)                                  # decimation over: the leaf all-reduce takes over
    assert not model.can_sum_gradients_at_scene_tensors(inp['imgs'])
