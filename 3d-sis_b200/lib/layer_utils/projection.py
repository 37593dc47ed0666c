"""Back-projection operators with the reference's interface (lib/layer_utils/projection.py):
`ProjectionHelper.compute_projection` and `Projection.apply`, on libsis3d kernels.

Host side: only the 4x4 inverses and the 8-corner frustum AABB (a few hundred flops per view, done
in fp32 torch-CPU ops in the reference's order so the cull bounds are bit-identical); the per-voxel
work (N0 = X*Y*Z transforms, projection, depth test, compaction) is on the GPU.
"""
import ctypes as C

import torch

from lib import _sis3d as S


def _corner_rays(intrinsic, image_dims, depth_min, depth_max):
    """Camera-space corner points of the view frustum, [8,4,1] (projection.py:16-19,27-38)."""
    w, h = image_dims
    pts = torch.ones(8, 4, 1, dtype=torch.float32)
    k = 0
    for d in (depth_min, depth_max):
        for ux, uy in ((0, 0), (w - 1, 0), (w - 1, h - 1), (0, h - 1)):
            x = (ux - intrinsic[0][2]) / intrinsic[0][0]
            y = (uy - intrinsic[1][2]) / intrinsic[1][1]
            pts[k, :3, 0] = torch.tensor([d * x, d * y, d], dtype=torch.float32)
            k += 1
    return pts


_CORNER_CACHE = {}


def view_params(intrinsic, image_dims, depth_min, depth_max, volume_dims, depths, poses, world2grid):
    """Pack the per-view constants consumed by sis3d_project_map: float32 [n,40] (CPU tensor).

    world_to_camera | grid_to_world | clamped frustum bounds (projection.py:56-60, 39-49), computed for
    all views in one batch of fp32 torch-CPU ops (bit-identical to the reference's per-view loop)."""
    # These are a handful of 4x4 products: keep them on the calling thread.  Letting torch fan tiny ops out
    # to its intra-op pool leaves dozens of spinning OpenMP workers behind, which on a CPU-quota'd
    # container (cgroup cpu.max) gets the whole process throttled for ~80 ms at a time (measured).
    nthreads = torch.get_num_threads()
    if nthreads > 1:
        torch.set_num_threads(1)
    try:
        return _view_params_impl(intrinsic, image_dims, depth_min, depth_max, volume_dims, poses, world2grid)
    finally:
        if nthreads > 1:
            torch.set_num_threads(nthreads)


def _view_params_impl(intrinsic, image_dims, depth_min, depth_max, volume_dims, poses, world2grid):
    poses = torch.as_tensor(poses, dtype=torch.float32).reshape(-1, 4, 4).cpu().contiguous()
    n = poses.shape[0]
    w2g = torch.as_tensor(world2grid, dtype=torch.float32).cpu().reshape(-1, 4, 4).contiguous()
    if w2g.shape[0] not in (1, n):
        raise S.Sis3dError("world2grid must be one matrix or one per view")
    # the reference's own inverses (projection.py:56-57); LAPACK handles each 4x4 of the batch independently
    inv = torch.inverse(torch.cat((poses, w2g))).contiguous()
    inv_p, inv_g = inv[:n], inv[n:]
    out = torch.empty(n, 40, dtype=torch.float32)
    S.check(S.lib.sis3d_view_params_host(C.c_void_p(poses.data_ptr()), C.c_void_p(w2g.data_ptr()), C.c_void_p(inv_p.data_ptr()),
                                         C.c_void_p(inv_g.data_ptr()), n, w2g.shape[0], C.c_double(intrinsic[0][0]),
                                         C.c_double(intrinsic[1][1]), C.c_double(intrinsic[0][2]), C.c_double(intrinsic[1][2]),
                                         int(image_dims[0]), int(image_dims[1]), C.c_double(depth_min), C.c_double(depth_max),
                                         int(volume_dims[0]), int(volume_dims[1]), int(volume_dims[2]),
                                         C.c_void_p(out.data_ptr())), "view_params_host")
    return out


def _view_params_torch(intrinsic, image_dims, depth_min, depth_max, volume_dims, poses, world2grid):
    """The same computation with the reference's torch ops (kept as the in-repo cross-check of the native helper)."""
    poses = torch.as_tensor(poses, dtype=torch.float32).reshape(-1, 4, 4).cpu()
    n = poses.shape[0]
    w2g = torch.as_tensor(world2grid, dtype=torch.float32).cpu().reshape(-1, 4, 4)
    if w2g.shape[0] == 1:
        w2g = w2g.expand(n, 4, 4).contiguous()
    corners = _corner_rays(intrinsic, image_dims, depth_min, depth_max)
    out = torch.zeros(n, 40, dtype=torch.float32)
    out[:, 0:16] = torch.inverse(poses).reshape(n, 16)
    out[:, 16:32] = torch.inverse(w2g).reshape(n, 16)
    c2w8 = poses[:, None].expand(n, 8, 4, 4).reshape(n * 8, 4, 4)
    g8 = w2g[:, None].expand(n, 8, 4, 4).reshape(n * 8, 4, 4)
    p = torch.bmm(c2w8, corners.repeat(n, 1, 1))
    pl = torch.round(torch.bmm(g8, torch.floor(p)))[:, :3, 0].reshape(n, 8, 3)
    pu = torch.round(torch.bmm(g8, torch.ceil(p)))[:, :3, 0].reshape(n, 8, 3)
    lo = torch.minimum(pl.min(1)[0], pu.min(1)[0])
    hi = torch.maximum(pl.max(1)[0], pu.max(1)[0])
    out[:, 32:35] = torch.clamp(lo, min=0)
    out[:, 35:38] = torch.minimum(hi, torch.tensor([float(v) for v in volume_dims], dtype=torch.float32))
    return out


def project_maps(views_dev, depths_dev, intr, cfgvals, volume_dims, img_w, img_h):
    """Launch sis3d_project_map for all views: returns (pix int16 [n,N0], counts int32 [n]) on device."""
    X, Y, Z = (int(v) for v in volume_dims)
    n = views_dev.shape[0]
    pix = torch.empty(n, X * Y * Z, dtype=torch.int16, device=views_dev.device)
    counts = torch.empty(n, dtype=torch.int32, device=views_dev.device)
    dmin, dmax, vs = cfgvals
    S.check(S.lib.sis3d_project_map(S.ptr(views_dev), S.ptr(depths_dev), n, img_w, img_h, S.f32(intr[0]), S.f32(intr[1]),
                                    S.f32(intr[2]), S.f32(intr[3]), S.f32(dmin), S.f32(dmax), S.f32(vs), X, Y, Z, S.ptr(pix), S.ptr(counts), S.stream()),
            "project_map")
    return pix, counts


class ProjectionHelper:
    def __init__(self, intrinsic, depth_min, depth_max, image_dims, volume_dims, voxel_size):
        self.intrinsic, self.depth_min, self.depth_max = intrinsic, depth_min, depth_max
        self.image_dims, self.volume_dims, self.voxel_size = image_dims, volume_dims, voxel_size

    def compute_projection(self, depth, camera_to_world, world_to_grid):
        """-> (lin_indices_3d, lin_indices_2d) int64 [N0+1] (element 0 = count) on the GPU, or None when no
        voxel projects validly (projection.py:52-121)."""
        dev = depth.device if depth.is_cuda else torch.device("cuda", torch.cuda.current_device())
        X, Y, Z = (int(v) for v in self.volume_dims)
        w, h = int(self.image_dims[0]), int(self.image_dims[1])
        vp = view_params(self.intrinsic, (w, h), self.depth_min, self.depth_max, (X, Y, Z), None,
                         camera_to_world, world_to_grid).to(dev)
        intr = (self.intrinsic[0][0], self.intrinsic[1][1], self.intrinsic[0][2], self.intrinsic[1][2])
        d = depth.to(dev, torch.float32).contiguous().reshape(1, h, w)
        pix, counts = project_maps(vp, d, intr, (self.depth_min, self.depth_max, self.voxel_size), (X, Y, Z), w, h)
        if int(counts[0].item()) == 0:
            return None
        n0 = X * Y * Z
        lin3d = torch.zeros(n0 + 1, dtype=torch.int64, device=dev)
        lin2d = torch.zeros(n0 + 1, dtype=torch.int64, device=dev)
        nbytes = int(S.lib.sis3d_project_compact_workspace_bytes(X, Y, Z))
        ws = torch.empty(max(nbytes, 8), dtype=torch.uint8, device=dev)
        S.check(S.lib.sis3d_project_compact(S.ptr(pix), X, Y, Z, S.ptr(lin3d), S.ptr(lin2d), S.ptr(ws),
                                            C.c_size_t(nbytes), S.stream()), "project_compact")
        return lin3d, lin2d


def backproject(feats, pix, pairs, n_pairs, volume_dims, img_w, img_h, feats_t=None):
    """feats [n,C,h,w] cuda -> VC volume [X,Y,Z,C] = max over paired views of (covered ? f : 0).  feats_t: where the
    channels-last copy of the features [n,h*w,C] goes (a new tensor when None)."""
    X, Y, Z = (int(v) for v in volume_dims)
    n, Cn = feats.shape[0], feats.shape[1]
    feats = feats.contiguous()
    if feats_t is None:
        feats_t = torch.empty(n, img_w * img_h, Cn, dtype=torch.float32, device=feats.device)
    vol = torch.empty(X, Y, Z, Cn, dtype=torch.float32, device=feats.device)
    S.check(S.lib.sis3d_backproject_max(S.ptr(feats), S.ptr(feats_t), S.ptr(pix), S.ptr(pairs), S.ptr(n_pairs), n, Cn,
                                        img_w, img_h, X, Y, Z, S.ptr(vol), S.stream()), "backproject_max")
    return vol


class Projection:
    """`Projection.apply(label, lin_indices_3d, lin_indices_2d, volume_dims)` -> [C,Z,Y,X]
    (projection.py:124-136); forward only."""

    @staticmethod
    def apply(label, lin_indices_3d, lin_indices_2d, volume_dims):
        dev = label.device
        if not label.is_cuda:
            raise S.Sis3dError("Projection.apply: CUDA tensors only")
        X, Y, Z = (int(v) for v in volume_dims)
        feat = label.float().reshape(1, -1, label.shape[-2], label.shape[-1]).contiguous()
        h, w = feat.shape[-2], feat.shape[-1]
        Cn = feat.shape[1]
        pad = (-Cn) % 4
        if pad:
            feat = torch.cat([feat, torch.zeros(1, pad, h, w, device=dev)], 1)
        l3 = lin_indices_3d.to(dev).contiguous().reshape(1, -1)
        l2 = lin_indices_2d.to(dev).contiguous().reshape(1, -1)
        pix = torch.empty(1, X * Y * Z, dtype=torch.int16, device=dev)
        S.check(S.lib.sis3d_project_scatter_lists(S.ptr(l3), S.ptr(l2), 1, X, Y, Z, S.ptr(pix), S.stream()), "scatter_lists")
        pairs = torch.zeros(3, dtype=torch.int32, device=dev)
        n_pairs = torch.ones(1, dtype=torch.int32, device=dev)
        vol = backproject(feat, pix, pairs, n_pairs, (X, Y, Z), w, h)
        return vol[..., :Cn].permute(3, 2, 1, 0).contiguous()
