"""FLAME decoder on the GPU: the drop-in for ``my_utils/photometric_optimization/models/FLAME.py`` (class ``FLAME``,
FLAME.py:36-216; ``FLAMETex``, FLAME.py:220-244) -- same constructor config, buffer names and ``forward`` signature /
return values -- with the linear blend skinning (``lbs``, models/lbs.py:141-228) running as two CUDA kernels
(``gifb200_flame_lbs``) instead of ~25 small torch ops.  SURVEY 8f.1: random FLAME parameters -> vertices -> rasteriser
-> shading -> condition map never leaves the device.

The landmark gathers (68 + 17 points) and the choice of the contour-landmark row (FLAME.py:88-132) stay as torch glue on
(B,)-sized tensors.  Inference only (the reference never differentiates through the decoder on the training path:
flame parameters come from the dataset)."""
import pickle

import numpy as np
import torch
import torch.nn as nn

from . import ops
from ._lib import check, lib, ptr, require_cuda, stream


def batch_rodrigues(rot_vecs):
    """models/lbs.py:247-279 (torch glue; used for the handful of neck-chain rotations only)."""
    angle = torch.norm(rot_vecs + 1e-8, dim=1, keepdim=True)
    d = rot_vecs / angle
    c, s = torch.cos(angle)[:, :, None], torch.sin(angle)[:, :, None]
    z = torch.zeros_like(d[:, 0])
    K = torch.stack([z, -d[:, 2], d[:, 1], d[:, 2], z, -d[:, 0], -d[:, 1], d[:, 0], z], 1).view(-1, 3, 3)
    return torch.eye(3, dtype=rot_vecs.dtype, device=rot_vecs.device)[None] + s * K + (1 - c) * (K @ K)


def vertices2landmarks(vertices, faces, lmk_faces_idx, lmk_bary_coords):
    """models/lbs.py:103-138."""
    B = vertices.shape[0]
    tri = faces[lmk_faces_idx]
    pts = vertices[torch.arange(B, device=vertices.device)[:, None, None], tri]
    return torch.einsum("blfi,blf->bli", pts, lmk_bary_coords)


def lbs(betas, pose, model):
    """``lbs`` of models/lbs.py:141-228 on a prepared model (see ``FLAME._prepare``): betas (B,NB), pose (B,NJ*3)
    axis-angle -> (verts (B,V,3), posed joints (B,NJ,3))."""
    betas, pose = betas.contiguous().float(), pose.contiguous().float()
    require_cuda(betas, pose)
    B, NB = betas.shape
    V, NJ = model["v_template"].shape[0], model["lbs_weights"].shape[1]
    if pose.shape != (B, NJ * 3) or NB != model["shapedirs_t"].shape[0]:
        raise ValueError(f"lbs: betas {tuple(betas.shape)} / pose {tuple(pose.shape)} do not match the model "
                         f"(NB={model['shapedirs_t'].shape[0]}, NJ={NJ})")
    verts = torch.empty(B, V, 3, device=betas.device)
    joints = torch.empty(B, NJ, 3, device=betas.device)
    nws = lib.gifb200_flame_lbs_workspace_bytes(B, NJ)
    ws = ops._workspace(nws, betas.device)
    check(lib.gifb200_flame_lbs(ptr(betas), ptr(pose), ptr(model["v_template"]), ptr(model["shapedirs_t"]),
                                ptr(model["posedirs"]), ptr(model["j_template"]), ptr(model["j_shapedirs"]),
                                ptr(model["parents_i32"]), ptr(model["lbs_weights"]), ptr(verts), ptr(joints), B, V, NB, NJ,
                                ptr(ws), nws, stream()), "gifb200_flame_lbs")
    return verts, joints


class FLAME(nn.Module):
    """Given FLAME parameters returns the mesh and the 2-D / 3-D landmark sets (reference FLAME.py:36-216)."""

    def __init__(self, config=None, arrays=None):
        super().__init__()
        if arrays is None:
            arrays = self._load_pickle(config)
        f32 = lambda a: torch.as_tensor(np.asarray(a), dtype=torch.float32) if not torch.is_tensor(a) else a.float()
        i64 = lambda a: torch.as_tensor(np.asarray(a), dtype=torch.long) if not torch.is_tensor(a) else a.long()
        self.dtype = torch.float32
        self.register_buffer("faces_tensor", i64(arrays["faces"]))
        self.register_buffer("v_template", f32(arrays["v_template"]).contiguous())
        self.register_buffer("shapedirs", f32(arrays["shapedirs"]).contiguous())           # (V,3,NB)  FLAME.py:53-55
        self.register_buffer("posedirs", f32(arrays["posedirs"]).contiguous())             # (P,3V)    FLAME.py:57-59
        self.register_buffer("J_regressor", f32(arrays["J_regressor"]).contiguous())
        parents = i64(arrays["parents"]).clone()
        parents[0] = -1
        self.register_buffer("parents", parents)
        self.register_buffer("lbs_weights", f32(arrays["lbs_weights"]).contiguous())
        self.register_parameter("eye_pose", nn.Parameter(torch.zeros(1, 6), requires_grad=False))     # FLAME.py:66-71
        self.register_parameter("neck_pose", nn.Parameter(torch.zeros(1, 3), requires_grad=False))
        for k in ("lmk_faces_idx", "dynamic_lmk_faces_idx", "full_lmk_faces_idx"):
            self.register_buffer(k, i64(arrays[k]))
        for k in ("lmk_bary_coords", "dynamic_lmk_bary_coords", "full_lmk_bary_coords"):
            self.register_buffer(k, f32(arrays[k]))
        chain, cur = [], 1                                                                   # FLAME.py:80-86
        while cur != -1:
            chain.append(cur)
            cur = int(self.parents[cur])
        self.register_buffer("neck_kin_chain", torch.tensor(chain, dtype=torch.long))
        # derived, kernel-side layouts (not part of the reference's state_dict)
        V, _, NB = self.shapedirs.shape
        self.register_buffer("shapedirs_t", self.shapedirs.permute(2, 0, 1).reshape(NB, V * 3).contiguous(), persistent=False)
        self.register_buffer("j_template", (self.J_regressor @ self.v_template).contiguous(), persistent=False)
        self.register_buffer("j_shapedirs", torch.einsum("jv,vkl->ljk", self.J_regressor, self.shapedirs)
                             .reshape(NB, -1).contiguous(), persistent=False)
        self.register_buffer("parents_i32", self.parents.to(torch.int32), persistent=False)

    @classmethod
    def from_arrays(cls, arrays):
        """Build from a dict of arrays (``gif_b200.flame_synth.synthetic_flame_model`` layout, or the fields of
        generic_model.pkl + landmark_embedding.npy already converted to dense arrays)."""
        return cls(arrays=arrays)

    @staticmethod
    def _load_pickle(config):
        """FLAME.py:44-78: generic_model.pkl (chumpy objects -> dense arrays) + landmark_embedding.npy."""
        with open(config.flame_model_path, "rb") as f:
            ss = pickle.load(f, encoding="latin1")
        dense = lambda a: np.array(a.todense() if "scipy.sparse" in str(type(a)) else a)
        shapedirs = dense(ss["shapedirs"])
        shapedirs = np.concatenate([shapedirs[:, :, :config.shape_params],
                                    shapedirs[:, :, 300:300 + config.expression_params]], 2)       # FLAME.py:54
        posedirs = dense(ss["posedirs"])
        emb = np.load(config.flame_lmk_embedding_path, allow_pickle=True, encoding="latin1")[()]
        return {"faces": dense(ss["f"]).astype(np.int64), "v_template": dense(ss["v_template"]), "shapedirs": shapedirs,
                "posedirs": np.reshape(posedirs, [-1, posedirs.shape[-1]]).T, "J_regressor": dense(ss["J_regressor"]),
                "parents": dense(ss["kintree_table"])[0].astype(np.int64), "lbs_weights": dense(ss["weights"]),
                "lmk_faces_idx": emb["static_lmk_faces_idx"], "lmk_bary_coords": emb["static_lmk_bary_coords"],
                "dynamic_lmk_faces_idx": np.asarray(emb["dynamic_lmk_faces_idx"]),
                "dynamic_lmk_bary_coords": np.asarray(emb["dynamic_lmk_bary_coords"]),
                "full_lmk_faces_idx": emb["full_lmk_faces_idx"], "full_lmk_bary_coords": emb["full_lmk_bary_coords"]}

    def _model(self):
        return {k: getattr(self, k) for k in ("v_template", "shapedirs_t", "posedirs", "j_template", "j_shapedirs",
                                              "parents_i32", "lbs_weights")}

    def _find_dynamic_lmk_idx_and_bcoords(self, pose, dynamic_lmk_faces_idx, dynamic_lmk_b_coords, neck_kin_chain,
                                          dtype=torch.float32):
        """FLAME.py:88-132: contour landmarks follow the head's y rotation relative to the neck chain."""
        B = pose.shape[0]
        aa = torch.index_select(pose.view(B, -1, 3), 1, neck_kin_chain)
        R = batch_rodrigues(aa.reshape(-1, 3)).view(B, -1, 3, 3)
        rel = torch.eye(3, device=pose.device, dtype=dtype)[None].expand(B, -1, -1)
        for i in range(len(neck_kin_chain)):
            rel = torch.bmm(R[:, i], rel)
        sy = torch.sqrt(rel[:, 0, 0] ** 2 + rel[:, 1, 0] ** 2)
        ang = torch.round(torch.clamp(torch.atan2(-rel[:, 2, 0], sy) * 180.0 / np.pi, max=39)).long()
        rows = torch.where(ang < 0, torch.where(ang < -39, torch.full_like(ang, 78), 39 - ang), ang)
        return dynamic_lmk_faces_idx[rows], dynamic_lmk_b_coords[rows]

    def seletec_3d68(self, vertices):
        """FLAME.py:169-173 (name as in the reference)."""
        B = vertices.shape[0]
        return vertices2landmarks(vertices, self.faces_tensor, self.full_lmk_faces_idx.repeat(B, 1),
                                  self.full_lmk_bary_coords.repeat(B, 1, 1))

    @torch.no_grad()
    def decode_vertices(self, shape_params, expression_params, pose_params, eye_pose_params=None):
        """The mesh only (what the conditioning render consumes): -> vertices (B,V,3), full pose (B,15)."""
        require_cuda(shape_params, expression_params, pose_params, eye_pose_params)
        B = shape_params.shape[0]
        if eye_pose_params is None:
            eye_pose_params = self.eye_pose.expand(B, -1)
        betas = torch.cat([shape_params, expression_params], dim=1)
        full_pose = torch.cat([pose_params[:, :3], self.neck_pose.expand(B, -1), pose_params[:, 3:], eye_pose_params], dim=1)
        return lbs(betas, full_pose, self._model())[0], full_pose

    @torch.no_grad()
    def forward(self, shape_params=None, expression_params=None, pose_params=None, eye_pose_params=None):
        """shape (B,n_shape), expression (B,n_exp), pose (B,6) = [global rotation | jaw] -> vertices (B,V,3),
        landmarks2d (B,68,3), landmarks3d (B,68,3)   (FLAME.py:175-216)."""
        vertices, full_pose = self.decode_vertices(shape_params, expression_params, pose_params, eye_pose_params)
        B = vertices.shape[0]
        dyn_idx, dyn_bc = self._find_dynamic_lmk_idx_and_bcoords(full_pose.float(), self.dynamic_lmk_faces_idx,
                                                                 self.dynamic_lmk_bary_coords, self.neck_kin_chain)
        idx = torch.cat([dyn_idx, self.lmk_faces_idx[None].expand(B, -1)], 1)
        bc = torch.cat([dyn_bc, self.lmk_bary_coords[None].expand(B, -1, -1)], 1)
        landmarks2d = vertices2landmarks(vertices, self.faces_tensor, idx, bc)
        return vertices, landmarks2d, self.seletec_3d68(vertices)


class FLAMETex(nn.Module):
    """FLAME.py:220-244: linear texture space (BFM-derived), texcode (B,n) -> albedo (B,3,256,256), BGR, in the units of
    the texture space (0..255 for FLAME_texture.npz).  ``gifb200_flametex`` evaluates the basis only at the texels the
    reference's nearest resize to 256 keeps, reading that part of the basis once per batch."""

    SIZE = 256

    def __init__(self, config=None, mean=None, basis=None):
        super().__init__()
        if mean is None:
            space = np.load(config.tex_space_path)
            mean, basis = space["mean"].reshape(1, -1), space["tex_dir"].reshape(-1, 200)[:, :config.tex_params]
        self.register_buffer("texture_mean", torch.as_tensor(np.asarray(mean), dtype=torch.float32).reshape(1, 1, -1))
        self.register_buffer("texture_basis", torch.as_tensor(np.asarray(basis), dtype=torch.float32)[None].contiguous())

    @torch.no_grad()
    def forward(self, texcode):
        texcode = texcode.float().contiguous()
        require_cuda(texcode, self.texture_basis)
        B, n = texcode.shape
        K = self.texture_mean.shape[-1]
        side = int(round((K // 3) ** 0.5))
        if side * side * 3 != K or self.texture_basis.shape[1:] != (K, n):
            raise ValueError(f"FLAMETex: texcode ({B}, {n}) does not match the texture space (mean {K}, basis "
                             f"{tuple(self.texture_basis.shape[1:])}, a square RGB texture)")
        out = torch.empty(B, 3, self.SIZE, self.SIZE, device=texcode.device)
        check(lib.gifb200_flametex(ptr(texcode), ptr(self.texture_mean), ptr(self.texture_basis), ptr(out), B, n, side,
                                   self.SIZE, stream()), "gifb200_flametex")
        return out
