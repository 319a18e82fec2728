"""GPU: the fused-loss step samples and scatters box-decimated textures at their cells (cell maps, DbwMapDesc.reserved) instead
of at the expanded atlases.  Same step both ways on the same seeded scene: the composited image and the loss must be identical
bit for bit, and every leaf gradient must agree to the rounding of the backward's atomics (which regroup the texture sums)."""
import pytest
import torch

from tests.test_model_gpu import _model_and_oracle, _inputs


def _step(model, inp, hard, cells):
    from dbw_b200.fused_loss import ScenePass, scene_mse
    st = model._static_arrays()
    (ev, ea, et), (bv, ba, bt, fmap, alpha) = model._scene_tensors(hard, cells=cells)
    assert (len(bt[0]) == 4 and bt[0][3] != 0) == cells
    env_pass = ScenePass(st['faces_e'], st['fvu_e'], st['fmap_e'], et, model.renderer_env, n_static_faces=model.bkg_n_faces)
    blk_pass = ScenePass(st['faces_b'], st['fvu_b'], st['fmap_b'], bt, model._phase()[2], alpha_group=model.alpha_group_faces or model.BNF)
    loss, rec = scene_mse(ev, ea, bv, ba, alpha, inp['R'], inp['T'], inp['imgs'], env_pass, blk_pass, fmap, return_rec=True)
    params = [q for q in model.parameters() if q.requires_grad]
    return loss.detach(), rec, torch.autograd.grad(loss, params, allow_unused=True)


@pytest.mark.gpu
def test_cell_maps_render_and_differentiate_like_the_atlases():
    model, tpl, p, dev = _model_and_oracle()
    inp, *_ = _inputs(dev)
    model._install_cameras(inp)
    assert model.training and model.is_live('decimate_txt') and model.decim_factor == 8
    _, hard, _ = model._phase()
    loss_a, rec_a, g_a = _step(model, inp, hard, cells=False)
    loss_c, rec_c, g_c = _step(model, inp, hard, cells=True)
    _, _, g_a2 = _step(model, inp, hard, cells=False)
    assert torch.equal(rec_a, rec_c) and torch.equal(loss_a, loss_c)
    names = [n for n, q in model.named_parameters() if q.requires_grad]
    for n, a, c, a2 in zip(names, g_a, g_c, g_a2):
        assert (a is None) == (c is None), n
        if a is None:
            continue
        scale = a.abs().max().item() + 1e-30
        spread = (a2 - a).abs().max().item() / scale                 # two runs of the same step: atomics in another order
        assert (c - a).abs().max().item() / scale <= max(1e-5, 4 * spread), (n, (c - a).abs().max().item() / scale, spread)
