"""CPU: a hard single-layer pass without opacities (the environment pass: K = 1, sigma = 0, save_fragment_state = 2) keeps no
fragment colours -- its backward has no opacity and no distance path, the colours' only use -- so its forward workspace is
smaller by exactly one 16 B colour per pixel.  Every other pass keeps them.  No kernel runs."""
import ctypes

import pytest
import torch

B, H, W = 3, 40, 56


def _align(x, a=256):
    return (x + a - 1) // a * a


def _settings(K, sigma, state):
    from dbw_b200.renderer import make_settings
    return make_settings(B, H, W, K, 30, 24, 2, 0, (2., 2., 0., 0.), sigma, 0. if sigma == 0 else 9.21 * sigma, 0.001,
                         (0, 0, 0), n_map_floats=2 * 8 * 8 * 3, save_fragment_state=state)


def _fwd_bytes(s):
    from dbw_b200 import _lib
    fwd, bwd = ctypes.c_size_t(0), ctypes.c_size_t(0)
    _lib.check(_lib.lib().dbw_workspace_bytes(ctypes.byref(s), ctypes.byref(fwd), ctypes.byref(bwd)), 'dbw_workspace_bytes')
    return fwd.value


def test_hard_single_layer_pass_without_opacities_keeps_no_colours():
    assert _fwd_bytes(_settings(1, 0., 1)) - _fwd_bytes(_settings(1, 0., 2)) == _align(B * H * W * 16)


@pytest.mark.parametrize('K, sigma', [(1, 1e-4), (10, 1e-4), (10, 0.)])
def test_other_passes_keep_their_colours(K, sigma):
    """sigma > 0 (a distance path), K = 10 (the blocks pass); opacities are save_fragment_state = 1 itself"""
    assert _fwd_bytes(_settings(K, sigma, 2)) == _fwd_bytes(_settings(K, sigma, 1))


def test_debug_hook_keeps_the_colours():
    from dbw_b200 import _lib
    L = _lib.lib()
    L.dbw_debug_keep_unread_outputs(1)
    try:
        kept = _fwd_bytes(_settings(1, 0., 2))
    finally:
        L.dbw_debug_keep_unread_outputs(0)
    assert kept == _fwd_bytes(_settings(1, 0., 1))


def test_scene_settings_declare_passes_without_opacities():
    from dbw_b200.renderer import scene_settings
    verts, faces = torch.zeros(12, 3), torch.zeros(20, 3, dtype=torch.int32)
    atlas, table = torch.zeros(8 * 8, 4), [(0, 8, 8)]
    args = (verts, faces, atlas, table, B, (2., 2., 0., 0.), (H, W))
    assert scene_settings(*args, 0., 1, maps_are_texels4=True)[0].save_fragment_state == 2
    assert scene_settings(*args, 0., 1, faces_alpha=torch.ones(20), maps_are_texels4=True)[0].save_fragment_state == 1
    with torch.no_grad():
        assert scene_settings(*args, 0., 1, maps_are_texels4=True)[0].save_fragment_state == 0


def test_opacities_are_refused_in_a_pass_declared_without_them():
    """the forward and the backward refuse faces_alpha under save_fragment_state = 2 (checked before any launch)"""
    from dbw_b200 import _lib
    L = _lib.lib()
    s = _settings(1, 0., 2)
    p = ctypes.c_void_p(256)                  # never dereferenced: the call fails on the settings first
    rc = L.dbw_render_forward(ctypes.byref(s), *([p] * 8), p, p, None, p, 1 << 30, None, None, None)
    assert rc != 0 and b'faces_alpha' in L.dbw_last_error()
    rc = L.dbw_render_backward(ctypes.byref(s), *([p] * 8), p, p, 1 << 30, p, None, p, p, p, None, None, p, 1 << 30, None)
    assert rc != 0 and b'faces_alpha' in L.dbw_last_error()
    s.save_fragment_state = 3
    rc = L.dbw_render_forward(ctypes.byref(s), *([p] * 8), None, p, None, p, 1 << 30, None, None, None)
    assert rc != 0 and b'save_fragment_state' in L.dbw_last_error()
