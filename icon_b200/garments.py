"""Garment extraction of the demo on the device: the `-seg_dir` step of apps/infer.py.

  extract_cloth   lib/common/cloth_extraction.py, called from apps/infer.py:566-605 once per garment of an image.
                  It cuts the reconstruction down to the faces whose vertices project into the garment's 2-D polygons,
                  less the body parts (hands, feet, head, and per DeepFashion2 category forearms, arms or legs) that
                  may overlap it.  The reference labels the vertices with an sklearn 1-NN classifier refitted per
                  garment and tests them with matplotlib's Path.contains_points; here both run in csrc/garments.cu
                  (icon_garment_labels, icon_garment_face_mask).

The polygon mapping (pinv of the projection) and the trimesh steps (Trimesh(recon.vertices, recon.faces),
update_faces, remove_unreferenced_vertices) stay on the host and are the reference's own calls, through the reference
module's globals; the device gives only the labels and the face mask.  Rules and arithmetic: DESIGN.md 4.16.

Cache: the reconstruction's vertices and faces, the SMPL vertices and the part table go to the device once, and the
labels are computed once, for as long as the next call passes equal arrays (compared element by element on the
host).  A different mesh, or the same object modified in place by any route, therefore never reuses stale labels;
the garments of one image share them.
"""
import json
import os

import numpy as np
import torch

from . import _C
from ._C import check, lib
from .ops import _p, _stream

REMOVE_ALWAYS = ("rightHand", "leftToeBase", "leftFoot", "rightFoot", "head", "leftHandIndex1", "rightHandIndex1",
                 "rightToeBase", "leftHand")
FOREARMS = ("leftForeArm", "rightForeArm")
ARMS = ("leftArm", "rightArm")
LEGS = ("leftLeg", "rightLeg")
MAX_PARTS = 32


def removed_parts(type_id):
    """Part names extract_cloth removes from a garment of DeepFashion2 category `type_id` (the reference's == tests)."""
    if type_id == 1 or type_id == 3 or type_id == 10:        # short sleeves
        return REMOVE_ALWAYS + FOREARMS
    if type_id == 5 or type_id == 6 or type_id == 12 or type_id == 13 or type_id == 8 or type_id == 9:
        return REMOVE_ALWAYS + FOREARMS + ARMS                # no sleeves, or lower-body clothes
    if type_id == 7:                                          # shorts
        return REMOVE_ALWAYS + LEGS + FOREARMS + ARMS
    return REMOVE_ALWAYS


def vertex_labels(recon_verts, smpl_verts, smpl_parts):
    """uint8 [V] on the device: the part id (smpl_parts: host array [S] of ids < 32) of each reconstruction vertex's
    nearest SMPL vertex, float64 rdist, lowest index on exact ties.  recon_verts [V,3] / smpl_verts [S,3]: float64
    CUDA tensors."""
    r, s = recon_verts.contiguous(), smpl_verts.contiguous()
    if r.dtype != torch.float64 or s.dtype != torch.float64 or r.dim() != 2 or r.shape[1] != 3 or s.dim() != 2 \
            or s.shape[1] != 3 or not (r.is_cuda and s.is_cuda):
        raise _C.IconError(f"vertex_labels: recon {tuple(r.shape)} {r.dtype} / smpl {tuple(s.shape)} {s.dtype} must "
                           "be float64 [N,3] CUDA tensors")
    parts = np.ascontiguousarray(smpl_parts, np.uint8)
    if parts.size != s.shape[0]:
        raise _C.IconError(f"vertex_labels: {parts.size} part ids for {s.shape[0]} SMPL vertices")
    out = torch.empty(r.shape[0], dtype=torch.uint8, device=r.device)
    with torch.cuda.device(r.device):
        nbytes = lib.icon_garment_labels_workspace_bytes(s.shape[0])
        ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=r.device)
        check(lib.icon_garment_labels(_p(r), r.shape[0], _p(s), s.shape[0], parts.ctypes.data, _p(out), _p(ws),
                                      nbytes, _stream()), "icon_garment_labels")
    return out


def face_mask(verts, faces, labels, remove_bits, polygons):
    """(mask uint8 [F], kept int32 [1]) on the device: the faces extract_cloth keeps.  verts [V,3] float64, faces
    [F,3] int64, labels [V] uint8 (CUDA tensors); remove_bits: bitmask of removed part ids; polygons: list of float64
    [n,2] host arrays, the garment's polygons already mapped to the reconstruction's x, y.  Synchronises."""
    v, f, lab = verts.contiguous(), faces.contiguous(), labels.contiguous()
    dev = v.device
    polys = [np.asarray(p, np.float64).reshape(-1, 2) for p in polygons]
    off = np.zeros(len(polys) + 1, np.int32)
    off[1:] = np.cumsum([len(p) for p in polys])
    xy = np.concatenate(polys) if polys else np.zeros((0, 2))
    xy_d = torch.from_numpy(np.ascontiguousarray(xy, np.float64)).to(dev)
    V, F = int(v.shape[0]), int(f.shape[0])
    mask = torch.empty(F, dtype=torch.uint8, device=dev)
    kept = torch.empty(1, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        nbytes = lib.icon_garment_face_mask_workspace_bytes(V, len(polys))
        ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
        check(lib.icon_garment_face_mask(_p(v), V, _p(f), F, _p(lab), int(remove_bits), _p(xy_d), len(xy),
                                         off.ctypes.data, len(polys), _p(mask), _p(kept), _p(ws), nbytes, _stream()),
              "icon_garment_face_mask")
    return mask, kept


def map_polygons(seg_coord, K, R, t, np_=np):
    """extract_cloth's polygon mapping, call for call: P = K[:3,:3] @ [R | t], XYZ = pinv(P) @ [x, y, 1] / XYZ[3];
    the 2-D polygons are XYZ[:, :2] (float64).  np_: the numpy the reference module imported."""
    extrinsic = np_.zeros((3, 4))
    extrinsic[:3, :3] = R
    extrinsic[:, 3] = t
    P = K[:3, :3] @ extrinsic
    P_inv = np_.linalg.pinv(P)
    polygons = []
    for polygon in seg_coord:
        n = len(polygon)
        coords_h = np_.hstack((polygon, np_.ones((n, 1))))
        XYZ = P_inv @ coords_h[:, :, None]
        XYZ = XYZ.reshape((XYZ.shape[0], XYZ.shape[1]))
        XYZ = XYZ[:, :3] / XYZ[:, 3, None]
        polygons.append(np.ascontiguousarray(XYZ[:, :2], np.float64))
    return polygons


def _read_part_table(path, n):
    """The reference's y table as (names, uint8 parts [n]), or None when the reference's own labelling would fail
    (a vertex no key lists, an index outside [0, n), more than MAX_PARTS keys)."""
    with open(path) as fh:
        table = json.load(fh)
    names = list(table.keys())
    if len(names) > MAX_PARTS:
        return None
    parts = np.full(n, -1, np.int64)
    for i, k in enumerate(names):
        idx = np.asarray(table[k])
        if idx.size and (idx.dtype.kind not in "iu" or idx.min() < 0 or idx.max() >= n):
            return None
        parts[idx.astype(np.int64)] = i
    if (parts < 0).any():
        return None
    return names, parts.astype(np.uint8)


class _Labels:
    """The device copies and labels of one (reconstruction, SMPL, part table), reused while the arrays are equal."""

    def __init__(self):
        self.host = None
        self.dev = None

    def get(self, recon_v, recon_f, smpl_v, parts, device):
        host = (recon_v, recon_f, smpl_v, parts)
        if self.host is not None and self.dev[0].device == device and all(
                a.shape == b.shape and np.array_equal(a, b) for a, b in zip(host, self.host)):
            return self.dev
        v = torch.from_numpy(recon_v).to(device)
        f = torch.from_numpy(recon_f).to(device)
        lab = vertex_labels(v, torch.from_numpy(smpl_v).to(device), parts)
        self.host = tuple(a.copy() for a in host)
        self.dev = (v, f, lab)
        return self.dev


def make_extract_cloth(reference_extract_cloth):
    """Overlay patch of lib.common.cloth_extraction: extract_cloth with the reference's signature and result.

    The polygons are mapped and the mesh is cut with the reference module's own numpy and trimesh, in the reference's
    order; the labels and the face mask come from the device.  Calls the device path cannot serve as the reference
    does go to `reference_extract_cloth` unchanged, and so return or raise what they do today: no SMPL body, a part
    table that leaves an SMPL vertex unlabelled (the SMPL-X body of -hps_type pixie), an empty or non-finite
    reconstruction or body, a non-finite mapped polygon vertex, or no CUDA device."""
    if reference_extract_cloth is None:
        raise _C.IconError("make_extract_cloth: the reference module has no extract_cloth")
    g = reference_extract_cloth.__globals__
    table_path = os.path.join(os.path.dirname(g["__file__"]), "smpl_vert_segmentation.json")
    cache = _Labels()

    def extract_cloth(recon, segmentation, K, R, t, smpl=None):
        if smpl is None or not torch.cuda.is_available():
            return reference_extract_cloth(recon, segmentation, K, R, t, smpl)
        recon_v = np.ascontiguousarray(recon.vertices, np.float64)
        recon_f = np.ascontiguousarray(recon.faces, np.int64)
        smpl_v = np.ascontiguousarray(smpl.vertices, np.float64)
        if recon_v.ndim != 2 or recon_v.shape[1] != 3 or len(recon_v) == 0 or smpl_v.ndim != 2 \
                or smpl_v.shape[1] != 3 or len(smpl_v) == 0 or not (np.isfinite(recon_v).all()
                                                                    and np.isfinite(smpl_v).all()):
            return reference_extract_cloth(recon, segmentation, K, R, t, smpl)
        table = _read_part_table(table_path, len(smpl_v))
        if table is None:
            return reference_extract_cloth(recon, segmentation, K, R, t, smpl)
        names, parts = table
        removed = removed_parts(segmentation["type_id"])
        if any(k not in names for k in removed):
            return reference_extract_cloth(recon, segmentation, K, R, t, smpl)

        mesh = g["trimesh"].Trimesh(recon.vertices, recon.faces)
        polygons = map_polygons(segmentation["coord_normalized"], K, R, t, g["np"])
        if not all(np.isfinite(p).all() for p in polygons):
            return reference_extract_cloth(recon, segmentation, K, R, t, smpl)

        dev = torch.device("cuda", torch.cuda.current_device())
        v, f, lab = cache.get(recon_v, recon_f, smpl_v, parts, dev)
        bits = 0
        for k in removed:
            bits |= 1 << names.index(k)
        mask_d, kept = face_mask(v, f, lab, bits, polygons)
        if int(kept.item()) == 0:
            return None
        mask = mask_d.cpu().numpy().astype(bool)
        mesh.update_faces(mask)
        mesh.remove_unreferenced_vertices()
        return mesh

    extract_cloth.__doc__ = make_extract_cloth.__doc__
    return extract_cloth
