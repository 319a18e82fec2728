"""oracle/dbw_path.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.  **PARITY UNPINNED** (see oracle/README.md).

CPU restatement (plain torch, fp32 or fp64, autograd for gradients) of the part of the render hot path the
reference itself owns, composed with the PyTorch3D restatement in oracle/pt3d.py:

    signed_pow                       <- src/utils/pytorch.py:31-32
    parametric_sq                    <- src/utils/superquadric.py:10-14
    point_to_uv_sphericalmap         <- src/utils/mesh.py:78-89
    get_icosphere / _uvs             <- src/utils/mesh.py:104-124, 127-169
    plane primitive                  <- primitives/plane.obj, src/utils/mesh.py:210-211
    elev/azim/roll rotation helpers  <- src/model/tools.py:173-207
    Renderer settings                <- src/model/renderer.py:24-60 (blur_radius = log(1/1e-4 - 1) * sigma, :51)
    LayeredShader.forward            <- src/model/renderer.py:219-238
    layered_rgb_blend                <- src/model/renderer.py:241-273
    _init_blocks / build_* / predict <- src/model/dbw.py:55-119, 202-239, 267-352
    rgb loss                         <- src/model/dbw.py:366-367 (nn.MSELoss via src/model/loss.py:15)

tests/golden/make_golden.py extracts the reference's own pure-torch functions with `ast` from a reference checkout and
stores their outputs under tests/golden/; tests/test_oracle_golden.py checks these restatements against them.
Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import this.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from . import pt3d

# ------------------------------------------------------------------ small math (utils/pytorch.py, superquadric.py)


def signed_pow(t, exponent):
    return torch.sign(t) * torch.abs(t).pow(exponent)


def parametric_sq(eta, omega, eps1, eps2):
    ce, se = signed_pow(torch.cos(eta), eps1), signed_pow(torch.sin(eta), eps1)
    co, so = signed_pow(torch.cos(omega), eps2), signed_pow(torch.sin(omega), eps2)
    return torch.stack([ce * so, se, ce * co], dim=-1)


def point_to_uv_sphericalmap(X, eps=1e-7):
    radius = torch.norm(X, dim=-1).clamp(min=eps)
    y = (X[..., 1] / radius).clamp(-1 + eps, 1 - eps)
    theta = torch.acos(-y)
    phi = torch.atan2(X[..., 0], X[..., 2])
    return torch.stack([(phi + np.pi) / (2 * np.pi), theta / np.pi], dim=-1)


def _axis_rotation(kind, deg):
    """tools.py:173-207: azim = angle with +X in the XZ plane, elev = angle with +Z in YZ, roll = angle with +X in XY."""
    a = float(deg) * np.pi / 180
    R = torch.eye(3)
    if kind == 'azim':
        c, s = math.cos(a), math.sin(a)
        R[0] = torch.tensor([c, 0., s]); R[2] = torch.tensor([-s, 0., c])
    elif kind == 'elev':
        c, s = math.cos(-a), math.sin(-a)
        R[1, 1:] = torch.tensor([c, s]); R[2, 1:] = torch.tensor([-s, c])
    else:
        c, s = math.cos(a), math.sin(a)
        R[0, :2] = torch.tensor([c, s]); R[1, :2] = torch.tensor([-s, c])
    return R


def world_rotation(elev, azim, roll):
    """dbw.py:58-59: R_world = elev @ azim @ roll, shape (1,3,3)."""
    return (_axis_rotation('elev', elev) @ _axis_rotation('azim', azim) @ _axis_rotation('roll', roll))[None]


# ------------------------------------------------------------------ topology / UV builders (utils/mesh.py)

def get_icosphere(level, flip_faces=False):
    verts, faces = pt3d.ico_sphere(level)
    if flip_faces:
        faces = torch.stack([faces[:, 2], faces[:, 1], faces[:, 0]], dim=-1)
    return verts, faces


def get_icosphere_uvs(level, fix_continuity=True, fix_poles=True, eps=1e-8):
    """Spherical UVs of the icosphere, with (i) faces that straddle the u seam re-pointed at duplicated UV verts
    shifted by +-1 and (ii) pole faces given their own pole UV vert at the mean u of the two other verts."""
    verts, faces = get_icosphere(level)
    verts_uvs = point_to_uv_sphericalmap(verts)
    if fix_continuity:
        vf = verts_uvs[faces]                                               # (F,3,2)
        du = torch.diff(vf[..., 0], dim=1, append=vf[..., 0:1, 0]).abs().max(1)[0]
        bad = du > 0.5
        bvf = vf[bad]
        u_c = bvf[..., 0] - 0.5 + eps
        side = torch.sign(u_c).sum(1)                                       # side holding 2 of the 3 verts
        lone = torch.sign(u_c) != side[:, None]
        new_u = bvf[..., 0] + side[:, None] * lone
        V = len(verts_uvs)
        extra = torch.stack([new_u[lone], bvf[..., 1][lone]], dim=-1)
        verts_uvs = torch.cat([verts_uvs, extra], 0)
        nf = faces.clone()
        ff = faces[bad].clone()
        ff[lone] = V + torch.arange(0, int(lone.sum()))
        nf[bad] = ff
        faces = nf
    if fix_poles:
        vf = verts_uvs[faces]
        bad = torch.logical_or(vf[..., 1].max(1)[0] > 0.99, vf[..., 1].min(1)[0] < 0.01)
        bvf = vf[bad]
        vv = bvf[..., 1]
        pole = torch.logical_or(vv > 0.99, vv < 0.01)
        u_mid = ((1 - pole.float()) * bvf[..., 0]).sum(1) / 2
        V = len(verts_uvs)
        extra = torch.stack([u_mid, vv[pole]], dim=-1)
        verts_uvs = torch.cat([verts_uvs, extra], 0)
        nf = faces.clone()
        ff = faces[bad].clone()
        ff[pole] = V + torch.arange(0, int(pole.sum()))
        nf[bad] = ff
        faces = nf
    return faces, verts_uvs


def get_plane():
    """primitives/plane.obj: 4 verts, 2 faces (1-based 'f 4 2 1' / 'f 4 3 2')."""
    verts = torch.tensor([[1., 0., -1.], [1., 0., 1.], [-1., 0., 1.], [-1., 0., -1.]])
    faces = torch.tensor([[3, 1, 0], [3, 2, 1]], dtype=torch.long)
    return verts, faces


def get_cube():
    """src/utils/mesh.py:172-173 (load_objs_as_meshes of primitives/cube.obj): 8 vertices of [-1,1]^3 and 12 triangles in
    the file's order; pinned against the file itself in tests/test_oracle_golden.py."""
    verts = torch.tensor([[1, -1, -1], [1, -1, 1], [-1, -1, 1], [-1, -1, -1], [1, 1, -1], [1, 1, 1], [-1, 1, 1], [-1, 1, -1]],
                         dtype=torch.float32)
    faces = torch.tensor([[1, 3, 0], [7, 5, 4], [4, 1, 0], [5, 2, 1], [2, 7, 3], [0, 7, 4], [1, 2, 3], [7, 6, 5], [4, 5, 1],
                          [5, 6, 2], [2, 6, 7], [0, 3, 7]], dtype=torch.long)
    return verts, faces


def get_cube_uvs():
    """src/utils/mesh.py:176-207: the unfolded-cross UV layout of the cube primitive."""
    faces_uvs = torch.tensor([[1, 3, 0], [7, 5, 4], [4, 9, 8], [11, 2, 10], [2, 7, 3], [12, 7, 13], [1, 2, 3], [7, 6, 5], [4, 5, 9],
                              [11, 6, 2], [2, 6, 7], [12, 3, 7]], dtype=torch.long)
    verts_uvs = torch.tensor([[0., 3 / 8], [0., 5 / 8], [1 / 4, 5 / 8], [1 / 4, 3 / 8], [3 / 4, 3 / 8], [3 / 4, 5 / 8], [2 / 4, 5 / 8],
                              [2 / 4, 3 / 8], [1., 3 / 8], [1., 5 / 8], [1 / 4, 7 / 8], [2 / 4, 7 / 8], [1 / 4, 1 / 8], [2 / 4, 1 / 8]],
                             dtype=torch.float32)
    return faces_uvs, verts_uvs


def cube_scene(texture, scale=0.5, R=None, T=None):
    """BASELINE configs[0]: ONE cube primitive with a (Ht,Wt,3) texture map in [0,1], posed by (v * scale) @ R + T."""
    verts, faces = get_cube()
    dt = texture.dtype
    verts = verts.to(dt) * scale
    if R is not None:
        verts = verts @ R.to(dt)
    if T is not None:
        verts = verts + T.to(dt)
    faces_uvs, verts_uvs = get_cube_uvs()
    return {'verts': verts, 'faces': faces, 'faces_verts_uvs': verts_uvs.to(dt)[faces_uvs],
            'face_map': torch.zeros(len(faces), dtype=torch.long), 'maps': [texture]}


# ------------------------------------------------------------------ renderer (renderer.py)

def blur_radius_from_sigma(sigma):
    return float(np.log(1. / 1e-4 - 1.) * sigma)


def layered_rgb_blend(colors, pix_to_face, dists, sigma, background=(0., 0., 0.), clip_inside=True, faces_alpha=None):
    """colors (N,H,W,K,3) -> (N,4,H,W).  Per-pixel front-to-back alpha compositing of the K z-sorted fragments,
    then the background; alpha channel = 1 - transmittance."""
    N, H, W, K = pix_to_face.shape
    bg = torch.as_tensor(background, dtype=colors.dtype)
    valid = (pix_to_face >= 0).to(colors)
    if sigma == 0:
        alpha = (dists <= 0).to(colors) * valid
    elif clip_inside:
        alpha = torch.exp(-dists.clamp(min=0) / sigma) * valid
    else:
        alpha = torch.sigmoid(-dists / sigma) * valid
    if faces_alpha is not None:
        alpha = alpha * faces_alpha.to(colors).gather(0, pix_to_face.reshape(-1).clamp(min=0)).view(alpha.shape)
    trans = torch.cumprod(1.0 - alpha, dim=-1)
    trans = torch.cat([torch.ones(N, H, W, 1, dtype=colors.dtype), trans], dim=-1)          # (N,H,W,K+1)
    colors_bg = torch.cat([colors, bg[None, None, None, None].expand(N, H, W, 1, -1)], dim=-2)
    alpha_bg = torch.cat([alpha, torch.ones(N, H, W, 1, dtype=colors.dtype)], dim=-1)
    rgb = (trans[..., None] * alpha_bg[..., None] * colors_bg).sum(-2)
    a = 1 - trans[..., -1]
    return torch.cat([rgb, a[..., None]], dim=-1).permute(0, 3, 1, 2)


def flat_shade_multiplier(verts, faces, R, direction=(1, 0.25, -1), ambient=(0.7, 0.7, 0.7), diffuse=(0.4, 0.4, 0.4)):
    """PyTorch3D flat_shading + DirectionalLights.diffuse for the reference's renderer_light (src/model/dbw.py:139-143):
    colour = (ambient + diffuse * relu(n_face . l)) * texel (+ specular 0); the reference re-expresses the light direction
    per view as direction @ R^T (src/model/renderer.py:87-89).  Returns (B,F,3)."""
    fv = verts[faces]
    n = F.normalize(torch.cross(fv[:, 1] - fv[:, 0], fv[:, 2] - fv[:, 0], dim=-1), p=2, dim=-1, eps=1e-6)
    d = torch.as_tensor(direction, dtype=verts.dtype)[None]
    l = F.normalize(d[None] @ R.to(verts.dtype).transpose(1, 2), p=2, dim=-1, eps=1e-6)      # (B,1,3)
    cos = torch.relu((n[None] * l).sum(-1))
    return torch.as_tensor(ambient, dtype=verts.dtype)[None, None] + torch.as_tensor(diffuse, dtype=verts.dtype)[None, None] * cos[..., None]


def render_edges(scene, R, T, K, image_size, linewidth=1, z_clip=None, faces_per_pixel=1):
    """Renderer.render_edges (src/model/renderer.py:134-146): K=1 hard rasterization, mask = -dists < (lw*2/min(size))^2."""
    verts_ndc = pt3d.world_to_ndc(scene['verts'], R, T, K)
    fr = pt3d.rasterize_meshes(verts_ndc, scene['faces'], image_size, blur_radius=0.0, faces_per_pixel=faces_per_pixel,
                               perspective_correct=True, clip_barycentric_coords=True, z_clip_value=z_clip)
    mask = (-fr.dists < (linewidth * 2 / min(image_size)) ** 2).to(verts_ndc)[:, None].max(-1)[0]
    return mask, fr.pix_to_face[..., 0]


def render(scene, R, T, K, image_size, sigma=1e-4, faces_per_pixel=25, z_clip=None, detach_bary=False,
           clip_inside=True, background=(0., 0., 0.), faces_alpha=None, perspective_correct=True, eps=1e-8,
           return_fragments=False, face_shade=None):
    """Renderer.forward (renderer.py:84-98) for the 'raw' LayeredShader: scene is a dict with
    verts (V,3), faces (F,3), faces_verts_uvs (F,3,2), face_map (F,), maps [ (Ht,Wt,3) ];
    R (B,3,3), T (B,3), K (4,4); faces_alpha None | (F,) | (B*F,) (batch-packed, dbw.py:219).  -> (B,4,H,W)."""
    B = R.shape[0]
    verts_ndc = pt3d.world_to_ndc(scene['verts'], R, T, K, eps=eps)
    frags = pt3d.rasterize_meshes(verts_ndc, scene['faces'], image_size, blur_radius=blur_radius_from_sigma(sigma),
                                  faces_per_pixel=faces_per_pixel, perspective_correct=perspective_correct,
                                  clip_barycentric_coords=True, cull_backfaces=False, z_clip_value=z_clip)
    if detach_bary:
        frags.bary_coords = frags.bary_coords.detach()
    texels = pt3d.sample_textures(frags, scene['faces_verts_uvs'], scene['face_map'], scene['maps'])
    if face_shade is not None:                      # (B,F,3) flat-shading multiplier, batch-packed like pix_to_face
        Fn = scene['faces'].shape[0]
        texels = texels * face_shade.reshape(-1, 3)[frags.pix_to_face.clamp(min=0)] * (frags.pix_to_face >= 0)[..., None]
    if faces_alpha is not None and faces_alpha.numel() == scene['faces'].shape[0]:
        faces_alpha = faces_alpha.repeat(B)
    out = layered_rgb_blend(texels, frags.pix_to_face, frags.dists, sigma, background, clip_inside, faces_alpha)
    return (out, frags) if return_fragments else out


# ------------------------------------------------------------------ scene construction (dbw.py)

def join_scenes(scenes):
    """join_meshes_as_scene: concatenate verts/faces (with offsets) and keep each map separately."""
    verts, faces, fvu, fmap, maps = [], [], [], [], []
    v_off = m_off = 0
    for s in scenes:
        verts.append(s['verts']); faces.append(s['faces'] + v_off)
        fvu.append(s['faces_verts_uvs']); fmap.append(s['face_map'] + m_off); maps += list(s['maps'])
        v_off += s['verts'].shape[0]; m_off += len(s['maps'])
    return {'verts': torch.cat(verts), 'faces': torch.cat(faces), 'faces_verts_uvs': torch.cat(fvu),
            'face_map': torch.cat(fmap), 'maps': maps}


class SceneTemplate:
    """Static topology of the DBW scene (dbw.py:55-96): background icosphere (level 2, flipped, radius z_far),
    ground plane (subdivided 3x), N block icospheres (level 1) with seam/pole-fixed UVs and circular u padding."""

    def __init__(self, n_blocks=10, S_world=0.5, R_world=(115, 0, 0), T_world=(0., 0., 0.), z_far=10,
                 ratio_block_scene=0.25, txt_size=256, txt_bkg_upscale=1, scale_min=0.2):
        self.n_blocks, self.S_world, self.z_far, self.ratio = n_blocks, S_world, z_far, ratio_block_scene
        self.txt_size, self.txt_bkg_upscale, self.scale_min = txt_size, txt_bkg_upscale, scale_min
        self.R_world = world_rotation(*R_world)
        self.T_world = torch.tensor(T_world, dtype=torch.float32)[None]
        bv, bf = get_icosphere(2, flip_faces=True)
        self.bkg_verts, self.bkg_faces = bv * z_far, bf
        self.bkg_verts_uvs = point_to_uv_sphericalmap(self.bkg_verts)
        gv, gf = get_plane()
        gv = gv * torch.tensor([z_far, 1, z_far], dtype=torch.float32)[None]
        for _ in range(3):
            gv, gf = pt3d.subdivide(gv, gf)
        self.ground_verts, self.ground_faces = gv, gf
        self.ground_verts_uvs = (gv[:, [0, 2]] / z_far + 1) / 2
        sv, sf = get_icosphere(1)
        self.block_faces = sf
        self.sq_eta = torch.asin(sv[..., 1])[None].expand(n_blocks, -1).clone()
        self.sq_omega = torch.atan2(sv[..., 0], sv[..., 2])[None].expand(n_blocks, -1).clone()
        faces_uvs, verts_uvs = get_icosphere_uvs(1, fix_continuity=True, fix_poles=True)
        p_left = abs(int(np.floor(verts_uvs.min(0)[0][0].item() * txt_size)))
        p_right = int(np.ceil((verts_uvs.max(0)[0][0].item() - 1) * txt_size))
        verts_u = (verts_uvs[..., 0] * txt_size + p_left) / (txt_size + p_left + p_right)
        self.block_verts_uvs = torch.stack([verts_u, verts_uvs[..., 1]], dim=-1)
        self.block_faces_uvs = faces_uvs
        self.txt_padding = (p_left, p_right)
        self.BNF = len(faces_uvs)

    def to_world(self, verts):
        return (verts * self.S_world) @ self.R_world.to(verts)[0] + self.T_world.to(verts)

    @staticmethod
    def _decimate(maps, factor):
        sub = F.avg_pool2d(maps.permute(0, 3, 1, 2), kernel_size=factor, stride=factor)
        return F.interpolate(sub, scale_factor=factor).permute(0, 2, 3, 1)

    def build_env(self, p, decimate=0):
        """join_meshes_as_scene([build_bkg(world_coord=True), build_ground(world_coord=True)]) (dbw.py:214,267-295)."""
        dt = p['texture_bkg'].dtype
        bkg_maps, ground_maps = torch.sigmoid(p['texture_bkg']), torch.sigmoid(p['texture_ground'])
        if decimate:
            bkg_maps, ground_maps = self._decimate(bkg_maps, decimate), self._decimate(ground_maps, decimate)
        bkg = {'verts': self.to_world(self.bkg_verts.to(dt)), 'faces': self.bkg_faces,
               'faces_verts_uvs': self.bkg_verts_uvs.to(dt)[self.bkg_faces],
               'face_map': torch.zeros(len(self.bkg_faces), dtype=torch.long), 'maps': [bkg_maps[0]]}
        gv = self.ground_verts.to(dt) @ pt3d.rotation_6d_to_matrix(p['R_6d_ground'])[0] + p['T_ground']
        ground = {'verts': self.to_world(gv), 'faces': self.ground_faces,
                  'faces_verts_uvs': self.ground_verts_uvs.to(dt)[self.ground_faces],
                  'face_map': torch.zeros(len(self.ground_faces), dtype=torch.long), 'maps': [ground_maps[0]]}
        return join_scenes([bkg, ground])

    def blocks_verts(self, p):
        eps1, eps2 = (torch.sigmoid(p['sq_eps']) * 1.8 + 0.1).split([1, 1], dim=-1)
        dt = p['sq_eps'].dtype
        return parametric_sq(self.sq_eta.to(dt), self.sq_omega.to(dt), eps1, eps2) * self.ratio

    def build_blocks(self, p, keep=None, decimate=0, alpha_noise=None):
        """build_blocks(as_scene=True) (dbw.py:297-346).  keep: bool mask of blocks to keep (opacity filter),
        alpha_noise: pre-drawn randn for the opacity noise.  Returns (scene or None, alpha of kept blocks)."""
        S = p['S'].exp() + self.scale_min
        Rm = pt3d.rotation_6d_to_matrix(p['R_6d'])
        logit = p['alpha_logit'] if alpha_noise is None else p['alpha_logit'] + alpha_noise
        alpha = torch.sigmoid(logit)
        maps = torch.sigmoid(p['textures'])
        verts = torch.bmm(self.blocks_verts(p) * S[:, None], Rm) + p['T'][:, None]
        if keep is not None:
            verts, maps, alpha = verts[keep], maps[keep], alpha[keep]
        NB = verts.shape[0]
        if NB == 0:
            return None, alpha
        if decimate:
            maps = self._decimate(maps, decimate)
        pl, pr = self.txt_padding
        maps = F.pad(maps.permute(0, 3, 1, 2), pad=(pl, pr, 0, 0), mode='circular').permute(0, 2, 3, 1)
        verts = self.to_world(verts)
        dt = verts.dtype
        fvu = self.block_verts_uvs.to(dt)[self.block_faces_uvs]
        scenes = [{'verts': verts[i], 'faces': self.block_faces, 'faces_verts_uvs': fvu,
                   'face_map': torch.zeros(self.BNF, dtype=torch.long), 'maps': [maps[i]]} for i in range(NB)]
        return join_scenes(scenes), alpha


def predict(tpl, p, R, T, K, image_size, sigma=1e-4, faces_per_pixel=10, z_clip=0.001, fine=False, keep=None,
            decimate=0, alpha_noise=None):
    """DifferentiableBlocksWorld.predict, decouple_rendering=True branch (dbw.py:213-223)."""
    env = tpl.build_env(p, decimate=decimate)
    rec_env = render(env, R, T, K, image_size, sigma=0, faces_per_pixel=1, z_clip=z_clip, detach_bary=False)[:, :3]
    blocks, alpha = tpl.build_blocks(p, keep=keep, decimate=decimate, alpha_noise=alpha_noise)
    if blocks is None:
        return rec_env * 1.0
    B = R.shape[0]
    faces_alpha = None if fine else alpha.repeat_interleave(tpl.BNF).repeat(B)
    out = render(blocks, R, T, K, image_size, sigma=sigma, faces_per_pixel=faces_per_pixel, z_clip=z_clip,
                 detach_bary=True, faces_alpha=faces_alpha)
    rec_fg, mask = out[:, :3], out[:, 3:]
    return rec_fg * mask + (1 - mask) * rec_env


def predict_joint(tpl, p, R, T, K, image_size, sigma=1e-4, faces_per_pixel=10, z_clip=0.001, fine=False, keep=None,
                  decimate=0, alpha_noise=None):
    """DifferentiableBlocksWorld.predict, decouple_rendering=False branch (dbw.py:225-232): background + ground + blocks as ONE
    scene through the (detach_bary) block renderer, environment faces at opacity 1."""
    env = tpl.build_env(p, decimate=decimate)
    blocks, alpha = tpl.build_blocks(p, keep=keep, decimate=decimate, alpha_noise=alpha_noise)
    scene = env if blocks is None else join_scenes([env, blocks])
    faces_alpha = None
    if not fine:
        n_env = env['faces'].shape[0]
        parts = [torch.ones(n_env, dtype=alpha.dtype)] + ([alpha.repeat_interleave(tpl.BNF)] if blocks is not None else [])
        faces_alpha = torch.cat(parts).repeat(R.shape[0])
    return render(scene, R, T, K, image_size, sigma=sigma, faces_per_pixel=faces_per_pixel, z_clip=z_clip, detach_bary=True,
                  faces_alpha=faces_alpha)[:, :3]


def safe_pow(t, exponent, eps=1e-6):
    """src/utils/pytorch.py:35-36"""
    return t.clamp(eps).pow(exponent)


def implicit_sq(points, eps1, eps2):
    """src/utils/superquadric.py:17-38 with safe=True, as_sdf=2 (the variant dbw.py:400 calls)"""
    points = points.clamp(-5, 5)
    x2, y2, z2 = [points[..., k].pow(2) for k in range(3)]
    x, y, z = safe_pow(x2, 1 / eps2), safe_pow(y2, 1 / eps1), safe_pow(z2, 1 / eps2)
    res = safe_pow(x + z, eps2 / eps1) + y
    return safe_pow(res, eps1 / 2) - 1


def regularisers(tpl, p, coarse=True, keep=None, tv_type='l2sq', unit_samples=None, weights=(1.0, 1.0, 1.0)):
    """the parameter-only terms of compute_losses (dbw.py:373-405): parsimony, total variation, overlap -> dict.
    keep: the kill_blocks / filter mask folded into _alpha_full (dbw.py:316-328); unit_samples: the U(0,1) draws of
    dbw.py:393 (N,1000,3), passed in so that both sides of a comparison use the same points."""
    tv_norm = {'l1': lambda t: t.abs().sum(-1), 'l2': lambda t: safe_pow(t.pow(2).sum(-1), 0.5), 'l2sq': lambda t: t.pow(2).sum(-1)}[tv_type]
    alpha_full = torch.sigmoid(p['alpha_logit'])
    if keep is not None:
        alpha_full = alpha_full * keep
    out = {}
    a = alpha_full if coarse else (alpha_full > 0.5).to(alpha_full)
    out['parsimony'] = weights[0] * (1 if coarse else 0) * safe_pow(a, 0.5).mean()
    factor = 1 if coarse else 0.1
    bkg, ground, blocks = torch.sigmoid(p['texture_bkg']), torch.sigmoid(p['texture_ground']), torch.sigmoid(p['textures'])
    tv = sum(tv_norm(torch.diff(bkg, dim=k)).mean() for k in (1, 2))
    dx = tv_norm(torch.diff(blocks, dim=2, append=blocks[:, :, 0:1]))
    dy = tv_norm(torch.diff(blocks, dim=1))
    tv = tv + dx.sum(0).mean() + dy.sum(0).mean()
    tv = tv + sum(tv_norm(torch.diff(ground, dim=k)).mean() for k in (1, 2)) * factor
    out['tv'] = weights[1] * factor * tv
    N = tpl.n_blocks
    S, Rm, T = p['S'].exp() + tpl.scale_min, pt3d.rotation_6d_to_matrix(p['R_6d']), p['T']
    eps1, eps2 = (torch.sigmoid(p['sq_eps']) * 1.8 + 0.1).split([1, 1], dim=-1)
    with torch.no_grad():
        pts = unit_samples.to(S) * 2 - 1
        pts = (pts * tpl.ratio * S[:, None]) @ Rm + T[:, None]
        pts = pts.reshape(-1, 3)[None].expand(N, -1, -1)
    inv = ((pts - T[:, None]) @ Rm.transpose(1, 2)) / (S[:, None] * tpl.ratio)
    occ = torch.sigmoid(-implicit_sq(inv, eps1, eps2) / 0.005) * a[:, None]
    out['overlap'] = weights[2] * (1 if coarse else 0) * (occ.sum(0) - 1.95).clamp(0).mean()
    return out


def mse_loss(imgs, rec):
    return ((imgs - rec) ** 2).mean()


# ------------------------------------------------------------------ synthetic inputs shared by tests and bench (SURVEY 8d)

def ring_cameras(n_views, dist=2.75, elev_deg=25.0, fx=4.8, dtype=torch.float32, jitter=0.0, seed=0):
    """n_views cameras on a ring looking at the origin, PyTorch3D convention X_cam = X_world @ R + T, shared K in
    the layout of src/dataset/dtu.py:102-106 (NDC focal fx, principal point 0)."""
    g = torch.Generator().manual_seed(seed)
    az = torch.arange(n_views, dtype=torch.float64) / max(n_views, 1) * 2 * math.pi
    el = torch.full((n_views,), elev_deg * math.pi / 180, dtype=torch.float64)
    if jitter:
        el = el + (torch.rand(n_views, generator=g, dtype=torch.float64) - 0.5) * jitter
    C = torch.stack([dist * torch.cos(el) * torch.sin(az), dist * torch.sin(el), dist * torch.cos(el) * torch.cos(az)], 1)
    zc = -C / C.norm(dim=1, keepdim=True)                     # camera +Z looks at the origin
    up = torch.tensor([0., 1., 0.], dtype=torch.float64)[None].expand(n_views, -1)
    xc = torch.cross(up, zc, dim=1); xc = xc / xc.norm(dim=1, keepdim=True)   # +X is left in PyTorch3D screen space
    yc = torch.cross(zc, xc, dim=1)
    R = torch.stack([xc, yc, zc], dim=2)                      # columns = camera axes (row-vector convention)
    T = -torch.bmm(C[:, None], R)[:, 0]
    Km = torch.zeros(4, 4, dtype=torch.float64)
    Km[0, 0] = Km[1, 1] = fx; Km[2, 3] = 1; Km[3, 2] = 1
    return R.to(dtype), T.to(dtype), Km.to(dtype)


def init_params(n_blocks=10, txt_size=256, txt_bkg_upscale=1, seed=227391, boxy=False, dtype=torch.float32,
                T_range=(1., 1., 1.), scale_min=0.2, opacity_init=0.5):
    """Parameter init of dbw.py:98-119 (random rotations drawn as normalised 6d vectors)."""
    g = torch.Generator().manual_seed(seed)
    N, TS, s = n_blocks, txt_size, txt_bkg_upscale
    p = {
        'sq_eps': torch.zeros(N, 2) if not boxy else (torch.rand(N, 2, generator=g) * 6 - 3),
        'R_6d_ground': torch.tensor([[1., 0., 0., 0., 1., 0.]]),
        'T_ground': torch.tensor([[0., -0.9 * T_range[1], 0.]]),
        'S': (torch.rand(N, 3, generator=g) + 0.5 - scale_min).log(),
        'R_6d': pt3d.matrix_to_rotation_6d(pt3d.rotation_6d_to_matrix(torch.randn(N, 6, generator=g))),
        'T': torch.randn(N, 3, generator=g) / 2 * torch.tensor(T_range),
        'alpha_logit': torch.logit(torch.ones(N) * opacity_init) + 1e-3,
        'texture_bkg': torch.randn(1, TS * s, TS * s, 3, generator=g) / 10,
        'texture_ground': torch.randn(1, TS * s, TS * s, 3, generator=g) / 10,
        'textures': torch.randn(N, TS, TS, 3, generator=g) / 10,
    }
    return {k: v.to(dtype) for k, v in p.items()}
