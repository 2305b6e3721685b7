"""Drop-in for reference `infer/wsi.py` (SURVEY.md row f2): `InferManager.process_wsi_list(run_args)` /
`process_single_file(wsi_path, msk_path, output_dir)` with the reference's run_args, patch / chunk /
tile geometry, tissue-mask patch selection, the three post-processing phases (grid tiles, boundary
strips, crosses) with their keep/replace merge rule and running-max id offsets, and the JSON output.

What changes underneath:
* patches go to the device in batches through `infer_step` (libhvn) and every tile through the device
  `process`; the reference's DataLoader workers and post-proc pool (`nr_inference_workers`,
  `nr_post_proc_workers`) are accepted and ignored;
* the WSI-sized prediction and instance maps live in host RAM (a disk memmap under `cache_path` only
  when they would not fit), not in `.npy` files that every stage re-opens (reference wsi.py:228,237,520-534);
* multi-GPU (one process per GPU, torch.distributed initialised): the patches of every chunk and the
  tiles of every phase are sharded across the ranks; per-patch maps are exchanged with one all_gather
  per chunk, per-tile results are gathered to rank 0, which alone applies the (order-dependent) merge
  callbacks in tile order and writes the JSON.  Tile results are merged in index order -- the order the
  reference produces with `nr_post_proc_workers=0` (with a pool its order is completion order).
* slides: `.npy` arrays and ordinary image files are read natively; OpenSlide formats need the
  `openslide` module (absent from this image) and raise a clear error otherwise.

Extension the reference lacks: run arg `save_features` (`run_infer.py wsi --save_features`) measures every nucleus of
every post-processing tile on the device (`_lib.FEATURE_NAMES`) on the tile's instance map, its region of the slide and
its prediction map, so each record carries "features" through the merge.  A nucleus cut by a tile edge is measured on
the same truncated pixels as its contour and bbox.  The merge never changes the pixels of a nucleus it keeps (a kept
old nucleus is left as it is, a new one is added only where it overlaps no kept one), so every written record's
features are those of its pixels in the final instance map.
"""
import glob
import logging
import os
import pathlib
import shutil
import time

import numpy as np

from . import base
from .tile import run_patches


def log_info(msg):
    logging.info(msg)


# ------------------------------------------------------------------------------------------------
# geometry (reference infer/wsi.py:64-221) -- all arguments are np.arrays in (y, x) order
def _get_patch_top_left_info(img_shape, input_size, output_size):
    """Top-left corners of the sliding windows (input) and of their centre regions (output):
    nr_step = floor((L - (in-out)) / out) + 1 windows per axis, step = out; x-major enumeration
    (np.meshgrid 'xy' indexing then flatten) -- reference wsi.py:64-88."""
    margin = input_size - output_size
    nr_step = np.floor((img_shape - margin) / output_size) + 1
    last = (margin // 2) + nr_step * output_size
    ys = np.arange(margin[0] // 2, last[0], output_size[0], dtype=np.int32)
    xs = np.arange(margin[1] // 2, last[1], output_size[1], dtype=np.int32)
    gy, gx = np.meshgrid(ys, xs)
    output_tl = np.stack([gy.flatten(), gx.flatten()], axis=-1)
    input_tl = output_tl - margin // 2
    return input_tl, output_tl


def _get_tile_info(img_shape, tile_shape, ambiguous_size=128):
    """The three tile sets of the post-processing: the grid (clipped to the image), the strips of
    +-ambiguous_size around every internal grid line, and the 4*ambiguous_size squares around every
    internal grid crossing -- reference wsi.py:92-151.  Each set is [n, 2 (tl, br), 2 (y, x)]."""
    grid_tl, _ = _get_patch_top_left_info(img_shape, tile_shape, tile_shape)
    grid_br = np.minimum(grid_tl + tile_shape, img_shape)
    tile_grid = np.stack([grid_tl, grid_br], axis=1)
    grid_x = np.unique(grid_tl[:, 1])
    grid_y = np.unique(grid_tl[:, 0])

    def coords(a, b):
        m = np.meshgrid(a, b)
        return np.stack([m[0].flatten(), m[1].flatten()], axis=-1)

    amb = ambiguous_size
    bx = np.stack([coords(grid_y, grid_x[1:] - amb), coords(grid_y + tile_shape[0], grid_x[1:] + amb)], axis=1)
    by = np.stack([coords(grid_y[1:] - amb, grid_x), coords(grid_y[1:] + amb, grid_x + tile_shape[1])], axis=1)
    tile_boundary = np.concatenate([bx, by], axis=0)
    tile_cross = np.stack([coords(grid_y[1:] - 2 * amb, grid_x[1:] - 2 * amb),
                           coords(grid_y[1:] + 2 * amb, grid_x[1:] + 2 * amb)], axis=1)
    return tile_grid, tile_boundary, tile_cross


def _get_chunk_patch_info(img_shape, chunk_input_shape, patch_input_shape, patch_output_shape):
    """Inference chunks and patches -- reference wsi.py:155-221.
    Returns chunk_info [n, 2 (in, out), 2 (tl, br), 2 (y, x)] and patch_info of the same layout.
    Kept quirk: a patch's *output* box is input_tl + (in - out), not + (in - out) // 2 (:181-182);
    it is only used for the mask selection."""
    def round_down(x, y):
        return np.floor(x / y) * y

    margin = patch_input_shape - patch_output_shape
    chunk_output_shape = round_down(chunk_input_shape - margin, patch_output_shape).astype(np.int64)
    chunk_input_shape = (chunk_output_shape + margin).astype(np.int64)

    p_in_tl, _ = _get_patch_top_left_info(img_shape, patch_input_shape, patch_output_shape)
    p_in_br = p_in_tl + patch_input_shape
    p_out_tl = p_in_tl + margin
    p_out_br = p_out_tl + patch_output_shape
    patch_info = np.stack([np.stack([p_in_tl, p_in_br], axis=1), np.stack([p_out_tl, p_out_br], axis=1)], axis=1)

    c_in_tl, _ = _get_patch_top_left_info(img_shape, chunk_input_shape, chunk_output_shape)
    c_in_br = c_in_tl + chunk_input_shape
    # chunks that stick out of the slide are shrunk to a whole number of patch outputs inside it
    for ax in (0, 1):
        sel = np.nonzero(c_in_br[:, ax] > img_shape[ax])[0]
        c_in_br[sel, ax] = (img_shape[ax] - margin[ax]) - c_in_tl[sel, ax]
        c_in_br[sel, ax] = round_down(c_in_br[sel, ax], patch_output_shape[ax])
        c_in_br[sel, ax] += c_in_tl[sel, ax] + margin[ax]
    c_out_tl = c_in_tl + margin // 2
    c_out_br = c_in_br - margin // 2
    chunk_info = np.stack([np.stack([c_in_tl, c_in_br], axis=1), np.stack([c_out_tl, c_out_br], axis=1)], axis=1)
    return chunk_info, patch_info


def _remove_inst(inst_map, remove_id_list):
    """Zero every instance whose id is listed (reference wsi.py:49-60), in one pass."""
    ids = np.asarray(list(remove_id_list))
    if ids.size:
        inst_map[np.isin(inst_map, ids)] = 0
    return inst_map


# ------------------------------------------------------------------------------------------------
# slide access (the role of reference misc/wsi_handler.py; the FileHandler protocol :12-92)
class ArrayHandler(object):
    """A slide held as an RGB array: `.npy` (memory-mapped) or an ordinary image file.  One
    magnification level (`base_mag`, default 40); other magnifications are produced by resizing like
    the reference does for levels a file lacks (wsi_handler.py:171-188)."""

    def __init__(self, file_path, base_mag=40.0):
        if str(file_path).endswith(".npy"):
            self.array = np.load(file_path, mmap_mode="r")
        else:
            import cv2
            img = cv2.imread(str(file_path))
            if img is None:
                raise IOError("cannot read slide %s" % file_path)
            self.array = cv2.cvtColor(img, cv2.COLOR_BGR2RGB)
        self.metadata = {"available_mag": [float(base_mag)], "base_mag": float(base_mag), "vendor": "array",
                         "mpp  ": None, "base_shape": np.array([self.array.shape[1], self.array.shape[0]])}
        self.image_ptr = None

    def get_dimensions(self, read_mag=None, read_mpp=None):
        """(x, y) at read_mag -- wsi_handler.py:49-57.  The reference truncates (its OpenSlide reader then resizes to that
        size); this handler's pixels come from cv2.resize(fx, fy), whose output size ROUNDS, so the shape is rounded the
        same way and always equals the array `read_region` serves."""
        scale = read_mag / self.metadata["base_mag"]
        return np.rint(self.metadata["base_shape"] * scale).astype(np.int32)

    def get_full_img(self, read_mag=None, read_mpp=None):
        import cv2
        scale = read_mag / self.metadata["base_mag"]
        img = np.asarray(self.array)[..., :3]
        if scale == 1.0:
            return img
        interp = cv2.INTER_CUBIC if scale > 1.0 else cv2.INTER_LINEAR
        return cv2.resize(img, (0, 0), fx=scale, fy=scale, interpolation=interp)

    def prepare_reading(self, read_mag=None, read_mpp=None, cache_path=None):
        self.image_ptr = self.array if read_mag == self.metadata["base_mag"] else self.get_full_img(read_mag=read_mag)

    def read_region(self, coords, size):
        """coords, size in (x, y) at the prepared magnification -- wsi_handler.py:139-164."""
        return np.array(self.image_ptr[coords[1] : coords[1] + size[1], coords[0] : coords[0] + size[0]])[..., :3]


def get_file_handler(path, backend):
    """reference misc/wsi_handler.py:191-203."""
    if backend in (".npy", ".png", ".jpg", ".jpeg", ".bmp"):
        return ArrayHandler(path)
    if backend in (".svs", ".tif", ".vms", ".vmu", ".ndpi", ".scn", ".mrxs", ".tiff", ".svslide", ".bif"):
        try:
            import openslide  # noqa: F401
        except ImportError:
            if backend in (".tif", ".tiff"):
                return ArrayHandler(path)
            raise ImportError("reading %s slides needs the `openslide` module; convert the slide to .npy "
                              "or install openslide-python" % backend)
        raise NotImplementedError("OpenSlide-backed reading is not wired up in this build")
    assert False, "Unknown WSI format `%s`" % backend


def simple_get_mask(wsi_thumb_rgb):
    """Tissue mask of a 1.25x thumbnail: Otsu threshold, drop dark specks < 256 px (8-connectivity),
    fill holes < 128*128 px, dilate by a radius-16 disk -- reference wsi.py:489-499, with
    scipy.ndimage / cv2 in the place of skimage.morphology (not installed here)."""
    import cv2
    from scipy import ndimage

    gray = cv2.cvtColor(wsi_thumb_rgb, cv2.COLOR_RGB2GRAY)
    _, mask = cv2.threshold(gray, 0, 255, cv2.THRESH_OTSU)
    mask = mask == 0
    eight = np.ones((3, 3), dtype=bool)
    lab, n = ndimage.label(mask, structure=eight)
    if n:
        sizes = np.bincount(lab.ravel())
        small = sizes < 16 * 16
        small[0] = False
        mask = mask & ~small[lab]
    # remove_small_holes(area_threshold): holes are background components (4-connectivity) of small area
    lab, n = ndimage.label(~mask)
    if n:
        sizes = np.bincount(lab.ravel())
        small = sizes < 128 * 128
        small[0] = False
        mask = mask | small[lab]
    r = 16
    yy, xx = np.mgrid[-r : r + 1, -r : r + 1]
    disk = (yy * yy + xx * xx <= r * r).astype(np.uint8)
    mask = cv2.dilate(mask.astype(np.uint8), disk) > 0
    return mask


# ------------------------------------------------------------------------------------------------
def _dist_info():
    try:
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized():
            return dist, dist.get_rank(), dist.get_world_size()
    except ImportError:
        pass
    return None, 0, 1


class InferManager(base.InferManager):
    """Run inference on whole-slide images."""

    # ---- stage 1: raw prediction ---------------------------------------------------------------
    def _select_valid_patches(self, patch_info_list, has_output_info=True):
        """Keep the boxes whose footprint in the tissue mask is non-empty (reference wsi.py:300-327)."""
        ratio = self.wsi_mask.shape[0] / self.wsi_proc_shape[0]
        keep = []
        for idx in range(patch_info_list.shape[0]):
            info = np.squeeze(patch_info_list[idx])
            box = np.rint((info[1] if has_output_info else info) * ratio).astype(np.int64)
            roi = self.wsi_mask[box[0][0] : box[1][0], box[0][1] : box[1][1]]
            if np.sum(roi) > 0:
                keep.append(idx)
        return patch_info_list[keep]

    def _get_raw_prediction(self, chunk_info_list, patch_info_list):
        """Every chunk: read it once, run its tissue patches through the network, write each patch's
        map into the slide-sized prediction map (reference wsi.py:329-383 + :237-260)."""
        win = self.patch_input_shape
        for idx in range(chunk_info_list.shape[0]):
            chunk_info = chunk_info_list[idx]
            start = chunk_info[0, 0]
            end = chunk_info[0, 1] - np.array(win)
            tl = patch_info_list[:, 0, 0]
            sel = (start[0] <= tl[:, 0]) & (tl[:, 0] <= end[0]) & (start[1] <= tl[:, 1]) & (tl[:, 1] <= end[1])
            chunk_patches = self._select_valid_patches(np.array(patch_info_list[sel]))
            if chunk_patches.shape[0] == 0:
                continue
            rel_tl = chunk_patches[:, 0, 0] - chunk_info[0, 0]  # patch input corner inside the chunk
            chunk_data = self.wsi_handler.read_region(chunk_info[0][0][::-1], (chunk_info[0][1] - chunk_info[0][0])[::-1])
            chunk_data = np.ascontiguousarray(np.array(chunk_data)[..., :3])
            pinfo = np.concatenate([rel_tl, np.zeros_like(rel_tl)], axis=1).astype(np.int64)
            outs = run_patches(chunk_data, pinfo, win[0], self.run_step, self.batch_size)
            out_tl = chunk_info[1][0]
            for (py, px), pdata in zip(rel_tl, outs):
                y0, x0 = int(out_tl[0] + py), int(out_tl[1] + px)
                self.wsi_pred_map[y0 : y0 + pdata.shape[0], x0 : x0 + pdata.shape[1]] = pdata
        return

    # ---- stage 2: post-processing --------------------------------------------------------------
    def _dispatch_post_processing(self, tile_info_list, callback):
        """Post-process every tile (sharded over the ranks) and feed the results to `callback` in tile
        order on rank 0 (reference wsi.py:385-437 with nr_post_proc_workers=0)."""
        dist, rank, world = _dist_info()
        nr_types = self.method["model_args"]["nr_types"]
        features = getattr(self, "save_features", False)
        if features:
            from ..models.hovernet.post_proc import process_features
        n = tile_info_list.shape[0]
        mine = []
        for idx in range(rank, n, world):
            tl, br = tile_info_list[idx][0], tile_info_list[idx][1]
            tile_pred = np.array(self.wsi_pred_map[tl[0] : br[0], tl[1] : br[1]])
            if features:  # with the tile's region of the slide, at the processing magnification
                region = np.ascontiguousarray(self.wsi_handler.read_region(tl[::-1], (br - tl)[::-1]))
                res = process_features(tile_pred, nr_types=nr_types, image=region)
            else:
                res = self.post_proc_func(tile_pred, nr_types=nr_types, return_centroids=True)
            mine.append((res, (idx, tl, br)))
        if world > 1:
            gathered = [None] * world if rank == 0 else None
            dist.gather_object(mine, gathered, dst=0)
            if rank != 0:
                return
            mine = sorted((r for part in gathered for r in part), key=lambda r: r[1][0])
        for res in mine:
            callback(res)
        return

    def _normal_tile_callback(self, args):
        """Phase 1 (reference wsi.py:569-604): shift to slide coordinates, offset ids by the running max."""
        (pred_inst, inst_info_dict), (_, tile_tl, tile_br) = args
        if len(inst_info_dict) == 0:
            return
        top_left = tile_tl[::-1]
        wsi_max_id = max(self.wsi_inst_info.keys()) if len(self.wsi_inst_info) > 0 else 0
        for inst_id, inst_info in inst_info_dict.items():
            inst_info["bbox"] += top_left
            inst_info["contour"] += top_left
            inst_info["centroid"] += top_left
            self.wsi_inst_info[inst_id + wsi_max_id] = inst_info
        pred_inst[pred_inst > 0] += wsi_max_id
        self.wsi_inst_map[tile_tl[0] : tile_br[0], tile_tl[1] : tile_br[1]] = pred_inst

    def _fixing_tile_callback(self, args):
        """Phases 2 and 3 (reference wsi.py:607-677): inside the strip / cross, keep the old nuclei that
        touch its edge, drop the old inner ones, and add the newly predicted nuclei that do not
        overlap a kept one."""
        (pred_inst, inst_info_dict), (_, tile_tl, tile_br) = args
        if len(inst_info_dict) == 0:
            return
        top_left = tile_tl[::-1]
        wsi_max_id = max(self.wsi_inst_info.keys()) if len(self.wsi_inst_info) > 0 else 0  # before the removal
        roi_inst = np.copy(self.wsi_inst_map[tile_tl[0] : tile_br[0], tile_tl[1] : tile_br[1]])
        roi_edge = np.concatenate([roi_inst[[0, -1], :].flatten(), roi_inst[:, [0, -1]].flatten()])
        roi_boundary_inst_list = np.unique(roi_edge)[1:]  # exclude background (reference :634; assumes a 0 on the edge)
        roi_inner_inst_list = np.unique(roi_inst)[1:]
        roi_inner_inst_list = np.setdiff1d(roi_inner_inst_list, roi_boundary_inst_list, assume_unique=True)
        roi_inst = _remove_inst(roi_inst, roi_inner_inst_list)
        self.wsi_inst_map[tile_tl[0] : tile_br[0], tile_tl[1] : tile_br[1]] = roi_inst
        for inst_id in roi_inner_inst_list:
            self.wsi_inst_info.pop(inst_id, None)

        overlap = pred_inst[roi_inst > 0]
        boundary_inst_list = np.unique(overlap)  # no background to exclude (reference :648)
        inner_inst_list = np.unique(pred_inst)[1:]
        inner_inst_list = np.setdiff1d(inner_inst_list, boundary_inst_list, assume_unique=True)
        pred_inst = _remove_inst(pred_inst, boundary_inst_list)
        for inst_id in inner_inst_list:
            if inst_id not in inst_info_dict:  # dropped by the < 3 contour points rule inside process
                log_info("Nuclei id=%d not in saved dict WRN1." % inst_id)
                continue
            inst_info = inst_info_dict[inst_id]
            inst_info["bbox"] += top_left
            inst_info["contour"] += top_left
            inst_info["centroid"] += top_left
            self.wsi_inst_info[inst_id + wsi_max_id] = inst_info
        pred_inst[pred_inst > 0] += wsi_max_id
        self.wsi_inst_map[tile_tl[0] : tile_br[0], tile_tl[1] : tile_br[1]] = roi_inst + pred_inst

    # ---- drivers -------------------------------------------------------------------------------
    def _parse_args(self, run_args):
        for variable, value in run_args.items():
            self.__setattr__(variable, value)
        self.chunk_shape = [self.chunk_shape, self.chunk_shape]
        self.tile_shape = [self.tile_shape, self.tile_shape]
        self.patch_input_shape = [self.patch_input_shape, self.patch_input_shape]
        self.patch_output_shape = [self.patch_output_shape, self.patch_output_shape]
        return

    def _alloc_map(self, name, shape, dtype):
        nbytes = int(np.prod(shape)) * np.dtype(dtype).itemsize
        try:
            import psutil
            fits = nbytes < 0.4 * psutil.virtual_memory().available
        except ImportError:
            fits = nbytes < (8 << 30)
        if fits:
            return np.zeros(shape, dtype=dtype)
        os.makedirs(self.cache_path, exist_ok=True)
        return np.lib.format.open_memmap("%s/%s.npy" % (self.cache_path, name), mode="w+", shape=tuple(shape), dtype=dtype)

    def process_single_file(self, wsi_path, msk_path, output_dir):
        """One slide -> `<output_dir>/[json/]<name>.json` (reference wsi.py:449-708)."""
        import cv2

        _, rank, _ = _dist_info()
        ambiguous_size = self.ambiguous_size
        tile_shape = np.array(self.tile_shape).astype(np.int64)
        chunk_input_shape = np.array(self.chunk_shape)
        patch_input_shape = np.array(self.patch_input_shape)
        patch_output_shape = np.array(self.patch_output_shape)

        path_obj = pathlib.Path(wsi_path)
        wsi_ext, wsi_name = path_obj.suffix, path_obj.stem

        start = time.perf_counter()
        self.wsi_handler = get_file_handler(wsi_path, backend=wsi_ext)
        self.wsi_proc_shape = self.wsi_handler.get_dimensions(self.proc_mag)
        self.wsi_handler.prepare_reading(read_mag=self.proc_mag, cache_path="%s/src_wsi.npy" % self.cache_path)
        self.wsi_proc_shape = np.array(self.wsi_proc_shape[::-1])  # to Y, X

        if msk_path is not None and os.path.isfile(msk_path):
            self.wsi_mask = cv2.imread(msk_path)
            self.wsi_mask = cv2.cvtColor(self.wsi_mask, cv2.COLOR_BGR2GRAY)
            self.wsi_mask[self.wsi_mask > 0] = 1
        else:
            log_info("WARNING: No mask found, generating mask via thresholding at 1.25x!")
            thumb = self.wsi_handler.get_full_img(read_mag=1.25)
            self.wsi_mask = np.array(simple_get_mask(thumb) > 0, dtype=np.uint8)
        if np.sum(self.wsi_mask) == 0:
            log_info("Skip due to empty mask!")
            return
        if rank == 0 and self.save_mask:
            cv2.imwrite("%s/mask/%s.png" % (output_dir, wsi_name), self.wsi_mask * 255)
        if rank == 0 and self.save_thumb:
            wsi_thumb_rgb = self.wsi_handler.get_full_img(read_mag=1.25)
            cv2.imwrite("%s/thumb/%s.png" % (output_dir, wsi_name), cv2.cvtColor(wsi_thumb_rgb, cv2.COLOR_RGB2BGR))

        out_ch = 3 if self.method["model_args"]["nr_types"] is None else 4
        self.wsi_inst_info = {}
        self.wsi_inst_map = self._alloc_map("pred_inst", tuple(self.wsi_proc_shape), np.int32) if rank == 0 else None
        self.wsi_pred_map = self._alloc_map("pred_map", tuple(self.wsi_proc_shape) + (out_ch,), np.float32)
        log_info("Preparing Input Output Placement: {0}".format(time.perf_counter() - start))

        start = time.perf_counter()
        chunk_info_list, patch_info_list = _get_chunk_patch_info(self.wsi_proc_shape, chunk_input_shape,
                                                                 patch_input_shape, patch_output_shape)
        self._get_raw_prediction(chunk_info_list, patch_info_list)
        log_info("Inference Time: {0}".format(time.perf_counter() - start))

        start = time.perf_counter()
        tile_grid_info, tile_boundary_info, tile_cross_info = _get_tile_info(self.wsi_proc_shape, tile_shape, ambiguous_size)
        tile_grid_info = self._select_valid_patches(tile_grid_info, False)
        tile_boundary_info = self._select_valid_patches(tile_boundary_info, False)
        tile_cross_info = self._select_valid_patches(tile_cross_info, False)
        self._dispatch_post_processing(tile_grid_info, self._normal_tile_callback)
        self._dispatch_post_processing(tile_boundary_info, self._fixing_tile_callback)
        self._dispatch_post_processing(tile_cross_info, self._fixing_tile_callback)
        log_info("Total Post Proc Time: {0}".format(time.perf_counter() - start))

        if rank != 0:
            return
        start = time.perf_counter()
        if self.save_mask or self.save_thumb:
            json_path = "%s/json/%s.json" % (output_dir, wsi_name)
        else:
            json_path = "%s/%s.json" % (output_dir, wsi_name)
        self._save_json(json_path, self.wsi_inst_info, mag=self.proc_mag)
        log_info("Save Time: {0}".format(time.perf_counter() - start))

    def process_wsi_list(self, run_args):
        """Every slide under run_args['input_dir'] (reference wsi.py:711-753)."""
        self.save_thumb = False
        self.save_mask = False
        self.save_features = False
        self.input_mask_dir = None
        self.cache_path = "cache"
        self._parse_args(run_args)
        dist, rank, world = _dist_info()
        if rank == 0:
            for sub, on in (("/json/", True), ("/thumb/", self.save_thumb), ("/mask/", self.save_mask)):
                if on and not os.path.exists(self.output_dir + sub):
                    os.makedirs(self.output_dir + sub)
        if world > 1:
            dist.barrier()
        wsi_path_list = glob.glob(self.input_dir + "/*")
        wsi_path_list.sort()  # ensure ordering
        for wsi_path in wsi_path_list[:]:
            if os.path.isdir(wsi_path):
                continue
            wsi_base_name = pathlib.Path(wsi_path).stem
            msk_path = "%s/%s.png" % (self.input_mask_dir, wsi_base_name)
            if self.save_thumb or self.save_mask:
                output_file = "%s/json/%s.json" % (self.output_dir, wsi_base_name)
            else:
                output_file = "%s/%s.json" % (self.output_dir, wsi_base_name)
            skip = os.path.exists(output_file)
            if world > 1:  # every rank must take the same branch (rank 0 writes the file mid-loop)
                flag = [skip]
                dist.broadcast_object_list(flag, src=0)
                skip = flag[0]
            if skip:
                log_info("Skip: %s" % wsi_base_name)
                continue
            try:
                log_info("Process: %s" % wsi_base_name)
                self.process_single_file(wsi_path, msk_path, self.output_dir)
                log_info("Finish")
            except Exception:
                if world > 1:
                    raise  # a rank that swallowed an error would leave the others waiting in a collective
                logging.exception("Crash")
        if os.path.isdir(self.cache_path):
            shutil.rmtree(self.cache_path, ignore_errors=True)
        return
