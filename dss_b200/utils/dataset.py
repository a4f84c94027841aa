"""``data_dict.npz`` of the multi-view reconstruction data (DSS/utils/dataset.py:30-211, written by
scripts/create_mvr_data_from_mesh.py:170-255): the cloud in object coordinates and one 4x4 world-to-view matrix per
image, plus the ground-truth image and mask files next to it (dataset.py:36-101: every file of ``<data_dir>/image`` /
``<data_dir>/mask`` with the configured extension, sorted; rgb -> (3,H,W) float32 in [0,1], mask -> (1,H,W) float 0/1),
read with PIL (the reference uses imageio, which this image lacks).  With ``load_dense_depth`` the dense depth maps
too (dataset.py:71-82, 204-209: every file of ``<data_dir>/<depth_folder>`` with ``depth_extension``, sorted; OpenEXR
through ``utils.io.read_exr``) -> (1,H,W) float32.  ``device_views`` uploads every view once into a
:class:`DeviceViews` store that the training loop gathers its batches from; ``pinned_batch`` stages a batch of views in
pinned host memory for a host->device copy."""
import copy
import os

import numpy as np
import torch

from ..core.camera import FoVPerspectiveCameras
from ..core.cloud import PointClouds3D

__all__ = ["MVRData", "DeviceViews", "decompose_to_R_and_t"]


def decompose_to_R_and_t(transform_mat, row_major=True):
    """4x4 transform -> R (..,3,3), t (..,3) in the row-vector convention X_view = X_world R + t
    (DSS/utils/mathHelper.py:163-174)."""
    if transform_mat.shape[-2:] != (4, 4):
        raise ValueError("Expecting batches of 4x4 matrices")
    if not row_major:
        transform_mat = transform_mat.transpose(-2, -1)
    return transform_mat[..., :3, :3], transform_mat[..., -1, :3]


class MVRData:
    """points / normals / colors and per-image ``camera_mat`` of a ``data_dict.npz``.

    ``data[i]`` -> ``{"camera_mat": (4,4) f32 [, "img.rgb": (3,H,W), "img.mask": (1,H,W), "img.depth": (1,H,W)]}``
    like ``MVRDataset.__getitem__`` (dataset.py:171-211); images are only present when given to the constructor, depth
    maps with ``load_dense_depth`` (or ``depths``, (H,W) arrays given by hand).  A count of depth maps other than the
    number of views, or a depth map of a size other than the images', is refused."""

    def __init__(self, data_dir_or_file, data_dict="data_dict.npz", images=None, masks=None, n_imgs=None,
                 img_folder="image", mask_folder="mask", img_extension="png", mask_extension="png", load_images=True,
                 load_dense_depth=False, depth_folder="depth", depth_extension="exr", depths=None):
        path = data_dir_or_file
        data_dir = None
        if os.path.isdir(path):
            data_dir = path
            path = os.path.join(path, data_dict)
        if load_images and data_dir is not None and images is None and masks is None:
            # dataset.py:41-57: the files of the two folders with the configured extension, sorted by name
            def listing(folder, ext):
                d = os.path.join(data_dir, folder)
                if not os.path.isdir(d):
                    return None
                return [os.path.join(d, f) for f in sorted(os.listdir(d)) if os.path.splitext(f)[1].lower()[1:] == ext]
            self.image_files, self.mask_files = listing(img_folder, img_extension), listing(mask_folder, mask_extension)
            if self.image_files:
                images = self.load_all_images()
            if self.mask_files:
                masks = self.load_all_masks()
        if load_dense_depth and depths is None:
            if data_dir is None:
                raise ValueError("load_dense_depth reads <data_dir>/%s: pass the data directory" % depth_folder)
            d = os.path.join(data_dir, depth_folder)
            if not os.path.isdir(d):
                raise ValueError("load_dense_depth: %s does not exist" % d)
            self.depth_files = [os.path.join(d, f) for f in sorted(os.listdir(d))
                                if os.path.splitext(f)[1].lower()[1:] == str(depth_extension).lower()]
            from .io import read_exr
            depths = [read_exr(f) for f in self.depth_files]
        self.data_dict = np.load(path, allow_pickle=True)
        if "camera_mat" not in self.data_dict:
            raise ValueError("data_dict must contain camera_mat!")
        self.camera_mat = np.asarray(self.data_dict["camera_mat"], dtype=np.float32)
        if self.camera_mat.ndim != 3 or self.camera_mat.shape[1:] != (4, 4):
            raise ValueError("camera_mat must be (n_images, 4, 4), got %s" % (self.camera_mat.shape,))
        for name, arr in (("images", images), ("masks", masks)):
            if arr is not None and len(arr) != len(self.camera_mat):
                raise ValueError("Found unequal number of %s and camera matrices! (%d, %d)"
                                 % (name, len(arr), len(self.camera_mat)))
        if depths is not None:
            if len(depths) != len(self.camera_mat):
                raise ValueError("Found invalid number of dense depth maps: %d for %d views"
                                 % (len(depths), len(self.camera_mat)))
            depths = [np.asarray(torch.as_tensor(d), dtype=np.float32).reshape(np.shape(d)[-2:]) for d in depths]
            size = None if images is None else tuple(torch.as_tensor(images[0]).shape[1:])
            for i, d in enumerate(depths):
                if d.shape != (size or depths[0].shape):
                    raise ValueError("depth map %d has size %s, but the images are %s" % (i, d.shape, size or depths[0].shape))
        self.images, self.masks, self.depths = images, masks, depths
        self.data_dir = data_dir          # None when a data_dict file was given: no mesh.obj to sample
        self._poisson_disk = {}           # get_pointclouds(num_points) samples, per count
        self.n_imgs = len(self.camera_mat) if n_imgs is None else min(int(n_imgs), len(self.camera_mat))

    def __len__(self):
        return self.n_imgs

    def load_all_images(self):
        """dataset.py:88-93: (3,H,W) float32 tensors in [0,1], alpha dropped."""
        from PIL import Image
        out = []
        for path in self.image_files:
            rgb = np.asarray(Image.open(path).convert("RGB"), dtype=np.float32) / 255.0
            out.append(torch.from_numpy(np.ascontiguousarray(rgb.transpose(2, 0, 1))))
        return out

    def load_all_masks(self):
        """dataset.py:95-101: 8-bit grey -> bool -> (1,H,W) float32 0/1."""
        from PIL import Image
        out = []
        for path in self.mask_files:
            m = np.asarray(Image.open(path).convert("L")).astype(bool)[None]
            out.append(torch.from_numpy(np.ascontiguousarray(m)).float())
        return out

    @property
    def resolution(self):
        return None if self.images is None else tuple(self.images[0].shape[1:])

    def pinned_batch(self, indices):
        """Views `indices` stacked in PINNED host memory, ready for one non-blocking copy per tensor:
        {"camera_mat": (B,4,4) [, "img.rgb": (B,3,H,W), "img.mask": (B,1,H,W)]} (what a training step uploads).
        An empty ``indices`` gives B = 0 tensors of the same trailing shapes and dtypes (a rank of a view-sharded
        step may be dealt no views)."""
        idx = [int(i) % len(self) for i in indices]
        pin = lambda t: t.pin_memory() if torch.cuda.is_available() else t
        out = {"camera_mat": pin(torch.from_numpy(self.camera_mat[np.asarray(idx, dtype=np.int64)]))}
        for key, arr in (("img.rgb", self.images), ("img.mask", self.masks)):
            if arr is None:
                continue
            if idx:
                out[key] = pin(torch.stack([torch.as_tensor(arr[i]) for i in idx]))
            else:
                first = torch.as_tensor(arr[0])
                out[key] = pin(first.new_empty((0,) + tuple(first.shape)))
        return out

    def device_views(self, device) -> "DeviceViews":
        """every view's image, mask, cameras and lights on ``device``, uploaded once (:class:`DeviceViews`)"""
        return DeviceViews(self, device)

    def __getitem__(self, idx):
        idx = idx % len(self)
        out = {"camera_mat": self.camera_mat[idx].copy()}
        if self.images is not None:
            out["img.rgb"] = self.images[idx]
        if self.masks is not None:
            out["img.mask"] = self.masks[idx]
        if self.depths is not None:
            out["img.depth"] = self.depths[idx][None]
        lights = self.data_dict["lights_%d" % idx] if ("lights_%d" % idx) in self.data_dict else None
        if lights is not None:
            props = lights.item() if hasattr(lights, "item") and lights.dtype == object else None
            if isinstance(props, dict):
                out["lights"] = {k: np.array(v, dtype=np.float32)[0] for k, v in props.items()
                                 if isinstance(v, (list, np.ndarray))}
        return out

    def light_props(self, device="cpu"):
        """``(light class, {property: (V, ...) tensor on device})`` of the views' own ``lights_%d`` entries: the class
        is ``PointLights`` when ``lights_type`` names it, else ``DirectionalLights``, and
        ``cls(**{k: v[idx] for k, v in props.items()})`` gives the lights of views ``idx``.  None when a view has no
        lights."""
        from ..core.lighting import DirectionalLights, PointLights
        lights = [self[i].get("lights") for i in range(len(self))]
        if any(l is None for l in lights):
            return None
        kind = str(self.data_dict["lights_type"]) if "lights_type" in self.data_dict else ""
        cls = PointLights if "PointLights" in kind else DirectionalLights
        vec = "location" if cls is PointLights else "direction"
        return cls, {k: torch.stack([torch.as_tensor(l[k]) for l in lights]).to(device)
                     for k in ("ambient_color", "diffuse_color", "specular_color", vec)}

    def get_pointclouds(self, num_points=None) -> PointClouds3D:
        """points, normals and colours in object coordinates (dataset.py:103-135).  With ``num_points`` None or the
        stored cloud's size, the stored cloud; otherwise ``num_points`` geodesic Poisson-disk samples of
        ``<data_dir>/mesh.obj`` (:func:`~dss_b200.ops.sample_points_poisson_disk`, seed 0, the reference's
        ``generate_sampling_poisson_disk(approximategeodesicdistance=True, exactnumflag=True)``) with colours of ones,
        on the CPU, computed on the current CUDA device once per count.  Raises ValueError when that file is missing."""
        t = lambda k: torch.tensor(np.asarray(self.data_dict[k]), dtype=torch.float32)
        points = t("points")
        if num_points is None or int(num_points) == points.shape[0]:
            colors = t("colors") if "colors" in self.data_dict else torch.ones_like(points)
            return PointClouds3D([points], [t("normals")], [colors])
        n = int(num_points)
        if n not in self._poisson_disk:
            mesh = self.sampled_mesh(n)
            from ..ops import sample_points_poisson_disk
            from .io import read_mesh
            verts, faces = read_mesh(mesh)
            dev = torch.device("cuda", torch.cuda.current_device())
            s = sample_points_poisson_disk(torch.from_numpy(verts).to(dev), torch.from_numpy(faces).to(dev), n,
                                           geodesic=True, seed=0)
            self._poisson_disk[n] = (s.points.cpu(), s.normals.cpu())
        p, nrm = self._poisson_disk[n]
        return PointClouds3D([p.clone()], [nrm.clone()], [torch.ones_like(p)])

    def sampled_mesh(self, num_points):
        """the path of ``<data_dir>/mesh.obj``, which ``get_pointclouds(num_points)`` samples; ValueError when it is
        missing (checked without sampling, so that a caller can refuse early)"""
        mesh = None if self.data_dir is None else os.path.join(self.data_dir, "mesh.obj")
        if mesh is None or not os.path.isfile(mesh):
            raise ValueError("get_pointclouds(%d) samples the data's mesh.obj, which %s" % (
                int(num_points), "a data_dict file has not" if mesh is None else "does not exist: %s" % mesh))
        return mesh

    def get_cameras(self, camera_mat=None, **camera_params):
        """``FoVPerspectiveCameras`` with R, T taken from ``camera_mat`` ((n,4,4) or (4,4); default: all images)
        (dataset.py:155-165; the stored ``cameras_params`` are used when present)."""
        params = dict(camera_params)
        if not params and "cameras_params" in self.data_dict:
            stored = self.data_dict["cameras_params"]
            stored = stored.item() if hasattr(stored, "item") else stored
            if isinstance(stored, dict):
                params = {k: v for k, v in stored.items() if k in ("znear", "zfar", "aspect_ratio", "fov", "degrees")}
        m = torch.as_tensor(self.camera_mat[:len(self)] if camera_mat is None else np.asarray(camera_mat), dtype=torch.float32)
        if m.dim() == 2:
            m = m[None]
        R, T = decompose_to_R_and_t(m)
        return FoVPerspectiveCameras(R=R.contiguous(), T=T.contiguous(), **params)


# float32 k / 255 for every byte k, correctly rounded: what load_all_images gives for an 8-bit value k
_BYTE_VALUES = np.arange(256, dtype=np.float32) / np.float32(255.0)


def _as_bytes(rgb, mask):
    """``(k, m)``: the bytes of one view, rgb (H,W,3) and mask (H,W) uint8, when every rgb value is bitwise some
    float32 k / 255 and every mask value +0 or 1; None otherwise"""
    if not np.isfinite(rgb).all():
        return None
    k = np.clip(np.rint(rgb * np.float32(255.0)), 0, 255).astype(np.uint8)
    if not np.array_equal(_BYTE_VALUES[k].view(np.uint32), rgb.view(np.uint32)):
        return None
    bits = mask.view(np.uint32)
    if not ((bits == 0) | (bits == np.float32(1.0).view(np.uint32))).all():
        return None
    return k.transpose(1, 2, 0), (bits != 0).astype(np.uint8)


class DeviceViews:
    """The views of an ``MVRData`` resident on one device, uploaded once, for the training loop and the validation
    (``MVRData.device_views(device)``).  V = ``len(data)`` views of H x W pixels:

    - ``store`` (V,H,W,4): r, g, b and mask per pixel.  uint8 when every rgb value is some float32 k / 255 and every
      mask value 0 or 1 (a data directory's 8-bit PNGs always are: 4 bytes per pixel), else float32 with the values'
      bits (images and masks passed to ``MVRData`` by hand, fractional masks included).  Never rounded.
    - ``camera_mat`` (V,4,4): the world-to-view matrices; ``proj`` (V,4,4): ``camera_matrices(data.get_cameras())``.
    - ``light_cls`` and ``light_props`` (``{property: (V,L,3)}``), as ``data.light_props`` gives them, or None when
      the data has no lights; :meth:`lights` selects views' lights from them.
    - ``depth`` (V,H,W) float32: the data's dense depth maps, or None without them; :meth:`depth_at` selects views.
    - ``nbytes``: the device bytes held.

    :meth:`batch` gives the training step's arguments for a list of views, the same bits as uploading
    ``data.pinned_batch``; ``ops.gather_views`` fills the images and masks from the store."""

    def __init__(self, data, device):
        from ..core.camera import camera_matrices
        if data.images is None or data.masks is None:
            raise ValueError("device_views needs the data's images and masks")
        self.device = torch.device(device)
        V = len(data)
        self.H, self.W = data.resolution
        rgb = [torch.as_tensor(data.images[i]).numpy() for i in range(V)]
        mask = [torch.as_tensor(data.masks[i]).numpy() for i in range(V)]
        for i in range(V):
            if rgb[i].dtype != np.float32 or rgb[i].shape != (3, self.H, self.W):
                raise TypeError("image %d must be a float32 (3, %d, %d) array, got %s %s"
                                % (i, self.H, self.W, rgb[i].dtype, rgb[i].shape))
            if mask[i].shape != (1, self.H, self.W):
                raise ValueError("mask %d must have shape (1, %d, %d), got %s" % (i, self.H, self.W, mask[i].shape))
            mask[i] = mask[i].astype(np.float32)[0]
        as_bytes = []
        for r, m in zip(rgb, mask):
            b = _as_bytes(r, m)
            if b is None:
                as_bytes = None
                break
            as_bytes.append(b)
        host = np.empty((V, self.H, self.W, 4), dtype=np.uint8 if as_bytes is not None else np.float32)
        for i in range(V):
            k, m = as_bytes[i] if as_bytes is not None else (rgb[i].transpose(1, 2, 0), mask[i])
            host[i, ..., :3], host[i, ..., 3] = k, m
        self.store = torch.from_numpy(host).to(self.device)
        self.camera_mat = torch.from_numpy(data.camera_mat[:V]).to(self.device)
        self.proj = camera_matrices(data.get_cameras())[0].to(self.device)
        lights = data.light_props(self.device)
        self.light_cls, self.light_props = (None, None) if lights is None else lights
        self.depth = None
        if data.depths is not None:
            self.depth = torch.from_numpy(np.stack(data.depths[:V])).to(self.device)
        held = [self.store, self.camera_mat, self.proj] + list((self.light_props or {}).values()) \
            + ([self.depth] if self.depth is not None else [])
        self.nbytes = sum(t.numel() * t.element_size() for t in held)

    def __len__(self):
        return self.store.shape[0]

    def check(self, idx):
        """the host list ``idx`` as view indices in [0, V): integers in [-V, V), taken % V as ``pinned_batch`` takes
        them; IndexError for any other value (the gather does not check its device indices)"""
        V = len(self)
        out = []
        for i in idx:
            j = int(i)
            if j != i or not -V <= j < V:
                raise IndexError("view index %r out of range for %d views" % (i, V))
            out.append(j % V)
        return out

    def upload(self, idx):
        """``idx`` (checked by :meth:`check`) as a (B,) int64 tensor on the device, copied without blocking from a
        fresh pinned tensor (the caching host allocator keeps it until the copy has run)"""
        t = torch.tensor(self.check(idx), dtype=torch.int64)
        if self.device.type == "cuda":
            t = t.pin_memory()
        return t.to(self.device, non_blocking=True)

    def gather(self, idx_dev, img=None, mask=None):
        """``(img (B,H,W,3), mask (B,H,W))`` float32 of the device indices ``idx_dev`` (``ops.gather_views``), into
        ``img`` / ``mask`` when given"""
        from ..ops import gather_views
        B = idx_dev.shape[0]
        if img is None:
            img = torch.empty((B, self.H, self.W, 3), dtype=torch.float32, device=self.device)
        if mask is None:
            mask = torch.empty((B, self.H, self.W), dtype=torch.float32, device=self.device)
        return gather_views(self.store, idx_dev, img, mask)

    def lights(self, idx_dev):
        """the lights of the device indices ``idx_dev``: ``light_cls`` with every property's rows ``idx_dev`` (what the
        training loop built from ``data.light_props``), or None without lights"""
        if self.light_cls is None:
            return None
        return self.light_cls(**{k: v.index_select(0, idx_dev) for k, v in self.light_props.items()},
                              device=self.device)

    def depth_at(self, idx_dev):
        """the (B,H,W) depth maps of the device indices ``idx_dev``; ValueError without depth maps"""
        if self.depth is None:
            raise ValueError("the views have no dense depth maps (MVRData(..., load_dense_depth=True))")
        return self.depth.index_select(0, idx_dev)

    def batch_at(self, idx_dev):
        """``(img, mask, proj, view, lights)`` of the device indices ``idx_dev``: the training step's arguments"""
        img, mask = self.gather(idx_dev)
        return (img, mask, self.proj.index_select(0, idx_dev), self.camera_mat.index_select(0, idx_dev),
                self.lights(idx_dev))

    def batch(self, idx):
        """``(img (B,H,W,3), mask (B,H,W), proj (B,4,4), view (B,4,4), lights)`` on the device for the host list
        ``idx`` (checked before anything is uploaded); an empty ``idx`` gives batch-0 tensors"""
        return self.batch_at(self.upload(idx))

    def check_rigid(self):
        """refuse with ValueError cameras the pose refinement cannot take (``ops.check_rigid_cameras``); checked once"""
        if not getattr(self, "_rigid", False):
            from ..ops import check_rigid_cameras
            check_rigid_cameras(self.camera_mat)
            self._rigid = True

    def with_poses(self, poses):
        """These views with every camera refined by ``poses`` (V,6), one correction per view (``ops.pose_cameras``):
        a ``DeviceViews`` sharing this one's store and lights, whose ``camera_mat`` and ``proj`` are the refined
        matrices of all V views (no gradient), so that ``evaluate_2d``, ``point_coverage`` and ``render_data_views``
        see the refined cameras.  Zero poses give this one's matrices bit for bit."""
        from ..ops import pose_cameras
        self.check_rigid()
        V = len(self)
        if tuple(poses.shape) != (V, 6):
            raise ValueError("poses must have shape (%d, 6), got %s" % (V, tuple(poses.shape)))
        out = copy.copy(self)
        with torch.no_grad():
            idx = torch.arange(V, dtype=torch.int64, device=self.device)
            out.camera_mat, out.proj = pose_cameras(poses.detach(), idx, self.camera_mat, self.proj)
        return out
