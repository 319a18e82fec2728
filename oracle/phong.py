"""float64 restatement of PyTorch3D's phong_shading as the reference's LayeredShader calls it (src/model/renderer.py:187-238):
Meshes.verts_normals_packed, the lights' diffuse / specular (pytorch3d/renderer/lighting.py), _apply_lighting and
phong_shading (pytorch3d/renderer/mesh/shading.py), over the fragments of `oracle.pt3d`, blended by the reference's
layered_rgb_blend.  Test infrastructure only.

PARITY UNPINNED, as for the rest of `oracle/pt3d.py`: PyTorch3D is not vendored, so these formulas restate its code and
defaults; nothing here is compared against PyTorch3D itself."""
import torch
import torch.nn.functional as F

from . import dbw_path as D
from . import pt3d

# PyTorch3D's defaults: DirectionalLights / PointLights, AmbientLights, Materials
LIGHT_DEFAULTS = {'ambient_color': (0.5, 0.5, 0.5), 'diffuse_color': (0.3, 0.3, 0.3), 'specular_color': (0.2, 0.2, 0.2),
                  'direction': (0., 1., 0.), 'location': (0., 1., 0.)}
MATERIAL_DEFAULTS = {'ambient_color': (1., 1., 1.), 'diffuse_color': (1., 1., 1.), 'specular_color': (1., 1., 1.), 'shininess': 64}


def vertex_normals(verts, faces):
    """Meshes.verts_normals_packed: index_add of (v2 - v1) x (v0 - v1) into each face's vertices, normalised (eps 1e-6)"""
    fv = verts[faces]
    fn = torch.cross(fv[:, 2] - fv[:, 1], fv[:, 0] - fv[:, 1], dim=1)
    n = torch.zeros_like(verts)
    for c in range(3):
        n = n.index_add(0, faces[:, c], fn)
    return F.normalize(n, eps=1e-6, dim=1)


def diffuse(normals, color, direction):
    """lighting.diffuse: color * relu(n . l), both normalised with eps 1e-6"""
    normals = F.normalize(normals, p=2, dim=-1, eps=1e-6)
    direction = F.normalize(direction, p=2, dim=-1, eps=1e-6)
    return color * torch.relu((normals * direction).sum(-1))[..., None]


def specular(points, normals, direction, color, camera_position, shininess):
    """lighting.specular: color * relu(v . reflect)^shininess, zero where n . l <= 0 (before the power)"""
    normals = F.normalize(normals, p=2, dim=-1, eps=1e-6)
    direction = F.normalize(direction, p=2, dim=-1, eps=1e-6)
    cos_angle = (normals * direction).sum(-1)
    mask = (cos_angle > 0).to(normals)
    view_direction = F.normalize(camera_position - points, p=2, dim=-1, eps=1e-6)
    reflect_direction = -direction + 2 * (cos_angle[..., None] * normals)
    alpha = torch.relu((view_direction * reflect_direction).sum(-1)) * mask
    return color * torch.pow(alpha, shininess)[..., None]


def light_terms(lights, materials, dtype=torch.float64):
    """(name, colours / vectors as float64 (3,) tensors, shininess) of the reference's lights kwargs and Materials kwargs"""
    lights, materials = dict(lights or {}), dict(materials or {})
    name = lights.get('name', 'ambient')
    vec = lambda v: torch.as_tensor(v, dtype=dtype).reshape(-1, 3)[0]
    L = {k: vec(lights.get(k, d)) for k, d in LIGHT_DEFAULTS.items()}
    if name == 'ambient':
        L['ambient_color'] = vec(lights.get('ambient_color', (1., 1., 1.)))
    M = {k: vec(materials.get(k, d)) for k, d in MATERIAL_DEFAULTS.items() if k != 'shininess'}
    return name, L, M, float(materials.get('shininess', MATERIAL_DEFAULTS['shininess']))


def phong_colors(frags, texels, verts, faces, R, T, lights=None, materials=None, normals=None):
    """phong_shading: (N,H,W,K,3) colours (ka La + kd diffuse) * texel + ks specular of the fragments of one scene seen by
    N = len(R) cameras (batch-packed pix_to_face n * F + f); a directional light re-expressed per view as direction @ R^T
    (renderer.py:87-89), the camera centre -T @ R^T"""
    name, L, M, shininess = light_terms(lights, materials, verts.dtype)
    normals = vertex_normals(verts, faces) if normals is None else normals
    p2f, bary = frags.pix_to_face, frags.bary_coords
    valid = (p2f >= 0)[..., None].to(bary)
    f = p2f.clamp(min=0) % faces.shape[0]
    # interpolate_face_attributes (empty slots -> 0)
    pts = (bary[..., None] * verts[faces][f]).sum(-2) * valid
    nrm = (bary[..., None] * normals[faces][f]).sum(-2) * valid
    ambient = M['ambient_color'] * L['ambient_color']
    if name == 'ambient':
        return ambient * texels
    B = R.shape[0]
    view = lambda t: t.reshape(B, 1, 1, 1, 3)
    cam = view(-(T[:, None].to(verts) @ R.to(verts).transpose(1, 2))[:, 0])
    if name == 'directional':
        direction = view(L['direction'][None, None] @ R.to(verts).transpose(1, 2))
    else:
        direction = L['location'] - pts
    d = diffuse(nrm, L['diffuse_color'], direction)
    s = specular(pts, nrm, direction, L['specular_color'], cam, shininess)
    return (ambient + M['diffuse_color'] * d) * texels + M['specular_color'] * s


def render_phong(scene, R, T, K, image_size, lights=None, materials=None, z_clip=None, faces_alpha=None, background=(0., 0., 0.),
                 perspective_correct=True, eps=1e-8):
    """the reference's Renderer(shading_type='phong', sigma=0, faces_per_pixel=1) forward: hard rasterization, phong_shading,
    layered_rgb_blend.  scene as dbw_path.render; K (4,4) / (1,4,4) shared, or (B,4,4) one per view.  -> (B,4,H,W)"""
    B = R.shape[0]
    Ks = K.reshape(-1, 4, 4)
    if len(Ks) > 1:                       # per-view intrinsics: one view at a time
        outs = []
        for b in range(B):
            fa = faces_alpha
            if fa is not None and fa.numel() == B * scene['faces'].shape[0]:
                fa = faces_alpha.reshape(B, -1)[b]
            outs.append(render_phong(scene, R[b:b + 1], T[b:b + 1], Ks[b], image_size, lights, materials, z_clip, fa, background,
                                     perspective_correct, eps))
        return torch.cat(outs)
    verts_ndc = pt3d.world_to_ndc(scene['verts'], R, T, Ks[0], eps=eps)
    frags = pt3d.rasterize_meshes(verts_ndc, scene['faces'], image_size, blur_radius=0.0, faces_per_pixel=1,
                                  perspective_correct=perspective_correct, clip_barycentric_coords=True, cull_backfaces=False,
                                  z_clip_value=z_clip)
    texels = pt3d.sample_textures(frags, scene['faces_verts_uvs'], scene['face_map'], scene['maps'])
    colors = phong_colors(frags, texels, scene['verts'], scene['faces'], R, T, lights, materials)
    if faces_alpha is not None and faces_alpha.numel() == scene['faces'].shape[0]:
        faces_alpha = faces_alpha.repeat(B)
    return D.layered_rgb_blend(colors, frags.pix_to_face, frags.dists, 0, background, True, faces_alpha)


def render_phong_viz(scene, R, T, K, image_size, **kw):
    """VizMeshRenderer's phong frame: render_phong at 4H x 4W, avg_pool2d(., 4)"""
    H, W = image_size
    return F.avg_pool2d(render_phong(scene, R, T, K, (4 * H, 4 * W), **kw), 4)
