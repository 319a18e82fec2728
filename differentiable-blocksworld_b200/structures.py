"""Host-side stand-ins for the PyTorch3D containers the reference passes through its render seam
(`Meshes`, `TexturesUV`, `join_meshes_as_scene`, `join_meshes_as_batch`; used at the reference's
src/model/dbw.py:74-96, 214-220, 260-265, 280, 295, 342-346).  They carry exactly what the CUDA kernels consume:
one vertex buffer, one int32 face buffer, per-face-vertex UVs, a per-face map index and the texture maps; nothing is
replicated per view (`extend(B)` only records B, it does not copy -- the reference's Meshes.extend + TexturesUV
replication is what forced its batch size down, SURVEY.md section 8 row a9)."""
import torch


class TexturesUV:
    """maps (N,H,W,3) | faces_uvs (N,F,3) long | verts_uvs (N,Vt,2); same constructor as
    pytorch3d.renderer.TexturesUV for the arguments the reference uses (dbw.py:280,295,342)."""

    def __init__(self, maps, faces_uvs, verts_uvs, align_corners=True, padding_mode='border', sampling_mode='bilinear'):
        assert align_corners and padding_mode == 'border' and sampling_mode == 'bilinear', \
            'only the sampling mode the reference uses is implemented (align_corners=True, border, bilinear)'
        if isinstance(maps, (list, tuple)):
            maps = torch.stack(list(maps)) if len(maps) else torch.zeros(0, 1, 1, 3)
        if isinstance(faces_uvs, (list, tuple)):
            faces_uvs = torch.stack(list(faces_uvs)) if len(faces_uvs) else torch.zeros(0, 0, 3, dtype=torch.long)
        if isinstance(verts_uvs, (list, tuple)):
            verts_uvs = torch.stack(list(verts_uvs)) if len(verts_uvs) else torch.zeros(0, 0, 2)
        # groups of same-sized maps; scene-level indexing
        self.map_groups = [maps] if maps.shape[0] > 0 else []
        self.faces_uvs = faces_uvs          # (N,F,3)
        self.verts_uvs = verts_uvs          # (N,Vt,2)
        self._scene = None                  # filled by join_scene: (faces_verts_uvs (F,3,2), face_map (F,))

    def __len__(self):
        return self.faces_uvs.shape[0]

    def maps_padded(self):
        assert len(self.map_groups) == 1
        return self.map_groups[0]

    def to(self, device):
        self.map_groups = [m.to(device) for m in self.map_groups]
        self.faces_uvs, self.verts_uvs = self.faces_uvs.to(device), self.verts_uvs.to(device)
        if self._scene is not None:
            self._scene = tuple(t.to(device) for t in self._scene)
        return self

    def n_maps(self):
        return sum(int(g.shape[0]) for g in self.map_groups)

    def scene_arrays(self):
        """(faces_verts_uvs (F,3,2) float, face_map (F,) int32) of the joined scene."""
        if self._scene is None:
            N, Fn = self.faces_uvs.shape[:2]
            idx = self.faces_uvs + (torch.arange(N, device=self.faces_uvs.device) * self.verts_uvs.shape[1])[:, None, None]
            fvu = self.verts_uvs.reshape(-1, 2)[idx.reshape(-1, 3)]
            fmap = torch.arange(N, device=fvu.device, dtype=torch.int32).repeat_interleave(Fn)
            self._scene = (fvu.contiguous(), fmap.contiguous())
        return self._scene

    def packed_maps(self):
        """All maps as one flat float buffer + [(offset, H, W)] per map (offsets in floats)."""
        table, off, flat = [], 0, []
        for g in self.map_groups:
            n, h, w, _ = g.shape
            for _ in range(n):
                table.append((off, h, w)); off += h * w * 3
            flat.append(g.reshape(-1))
        return (flat[0] if len(flat) == 1 else torch.cat(flat)), table

    @staticmethod
    def join_scene(textures):
        """Scene-level texture of several TexturesUV (each possibly holding several meshes)."""
        out = TexturesUV.__new__(TexturesUV)
        out.map_groups, fvus, fmaps, m_off = [], [], [], 0
        for t in textures:
            fvu, fmap = t.scene_arrays()
            fvus.append(fvu); fmaps.append(fmap + m_off)
            out.map_groups += list(t.map_groups); m_off += t.n_maps()
        out._scene = (torch.cat(fvus), torch.cat(fmaps))
        out.faces_uvs = torch.zeros(1, out._scene[0].shape[0], 3, dtype=torch.long)
        out.verts_uvs = torch.zeros(1, 0, 2)
        return out


class Meshes:
    """A batch of N meshes with identical vertex/face counts: verts (N,V,3), faces (N,F,3) long."""

    def __init__(self, verts, faces, textures=None):
        if isinstance(verts, (list, tuple)):
            verts = torch.stack(list(verts)) if len(verts) else torch.zeros(0, 0, 3)
        if isinstance(faces, (list, tuple)):
            faces = torch.stack(list(faces)) if len(faces) else torch.zeros(0, 0, 3, dtype=torch.long)
        self._verts, self._faces, self.textures = verts, faces, textures
        self._n_views = None          # set by extend(): the same scene seen by B cameras

    def __len__(self):
        return self._verts.shape[0] if self._n_views is None else self._n_views

    @property
    def device(self):
        return self._verts.device

    def to(self, device):
        self._verts, self._faces = self._verts.to(device), self._faces.to(device)
        if self.textures is not None:
            self.textures = self.textures.to(device)
        return self

    def verts_padded(self):
        return self._verts

    def faces_padded(self):
        return self._faces

    def verts_packed(self):
        return self._verts.reshape(-1, 3)

    def faces_packed(self):
        N, Fn = self._faces.shape[:2]
        off = (torch.arange(N, device=self._faces.device) * self._verts.shape[1])[:, None, None]
        return (self._faces + off).reshape(-1, 3)

    def get_mesh_verts_faces(self, i):
        return self._verts[i], self._faces[i]

    def num_faces_per_mesh(self):
        return torch.full((self._faces.shape[0],), self._faces.shape[1], dtype=torch.long)

    def scale_verts(self, s):
        return Meshes(self._verts * s, self._faces, self.textures)

    def scale_verts_(self, s):
        self._verts = self._verts * s
        return self

    def extend(self, B):
        """The reference replicates the scene B times (dbw.py:215,220); here it is a view that records B."""
        assert self._verts.shape[0] == 1, 'extend() expects a single (joined) scene mesh'
        out = Meshes(self._verts, self._faces, self.textures)
        out._n_views = int(B)
        return out


def join_meshes_as_batch(meshes):
    return Meshes(torch.cat([m.verts_padded() for m in meshes]), torch.cat([m.faces_padded() for m in meshes]))


def join_meshes_as_scene(meshes):
    """One mesh holding every vertex/face of the inputs (a Meshes batch or a list of Meshes)."""
    if isinstance(meshes, Meshes):
        meshes = [meshes]
    verts = torch.cat([m.verts_packed() for m in meshes])
    faces, off = [], 0
    for m in meshes:
        faces.append(m.faces_packed() + off); off += m.verts_packed().shape[0]
    txt = None
    if all(m.textures is not None for m in meshes):
        txt = TexturesUV.join_scene([m.textures for m in meshes])
    return Meshes(verts[None], torch.cat(faces)[None], txt)
