"""Drop-in for reference `infer/tile.py` (SURVEY.md row f1): `InferManager.process_file_list(run_args)`
with the reference's run_args, patch geometry, stitching, and `.mat` / `.json` / overlay / QuPath outputs.

What changes underneath: patches go to the device in batches through libhvn, the stitched maps are post-processed by
the device `process` in this process (the reference's `nr_post_proc_workers` pool and `nr_inference_workers` loader
processes are accepted and ignored -- there is no CPU stage left to parallelise).  Files are cached in groups by the
reference's RAM budget (`mem_usage` of the available RAM, `sys.getsizeof(padded image) * 5` per file), further bounded
by half of the free device memory; the patches of a whole group run as one stream of `batch_size` batches that span
image boundaries (`hvn_infer_tiles`), and equal-size images are post-processed together.  On one GPU a group runs on
the device while the previous group's files are written and the next group's files are read.  Unlike the reference, a
file that exceeds the budget on its own is processed as a group of one instead of being skipped.

Extension the reference lacks: run arg `save_features` (`run_infer.py tile --save_features`) measures every nucleus on the
device (`_lib.FEATURE_NAMES`: shape, colour and NP-probability statistics, hvn_inst_features) before the group's device
maps are freed.  The JSON records gain "features" and the `.mat` gains `inst_features` [n,18] (rows in `inst_uid`
order) and `inst_feature_names`."""
import glob
import math
import os
import pathlib
import re
import shutil
import sys

import numpy as np

from . import base


def _prepare_patching(img, window_size, mask_size, return_src_top_corner=False):
    """Reflect-pad `img` and list the patch grid: rows of (y, x, row_idx, col_idx) in the padded image.
    Geometry of reference infer/tile.py:46-94: step = mask_size; last = (ceil((L-mask)/step)+1)*step;
    pad top/left = (window-mask)//2, pad bottom/right = last + window - L."""
    win, step = int(window_size), int(mask_size)
    im_h, im_w = img.shape[0], img.shape[1]

    def last_step(length):
        return int((math.ceil((length - step) / step) + 1) * step)

    last_h, last_w = last_step(im_h), last_step(im_w)
    padt = padl = (win - step) // 2
    padb, padr = last_h + win - im_h, last_w + win - im_w
    img = np.pad(img, ((padt, padb), (padl, padr), (0, 0)), "reflect")
    ys = np.arange(0, last_h, step, dtype=np.int32)
    xs = np.arange(0, last_w, step, dtype=np.int32)
    # the reference enumerates x-major (meshgrid default 'xy' indexing, then flatten)
    gy, gx = np.meshgrid(ys, xs)
    ry, rx = np.meshgrid(np.arange(ys.size, dtype=np.int32), np.arange(xs.size, dtype=np.int32))
    patch_info = np.stack([gy.flatten(), gx.flatten(), ry.flatten(), rx.flatten()], axis=-1)
    if return_src_top_corner:
        return img, patch_info, [padt, padl]
    return img, patch_info


def _stitch(patch_info, patch_data, src_shape):
    """Re-assemble per-patch outputs [n,h,w,C] into the map of the source image (reference
    infer/tile.py:110-131): sort by (y, x), tile as rows x cols, crop to the source shape."""
    order = sorted(range(len(patch_info)), key=lambda i: (int(patch_info[i][0]), int(patch_info[i][1])))
    info = [patch_info[i] for i in order]
    data = np.stack([patch_data[i] for i in order])
    nr_row = max(int(p[2]) for p in info) + 1
    nr_col = max(int(p[3]) for p in info) + 1
    ph, pw, ch = data.shape[1:]
    m = data.reshape(nr_row, nr_col, ph, pw, ch).transpose(0, 2, 1, 3, 4).reshape(nr_row * ph, nr_col * pw, ch)
    return np.ascontiguousarray(m[: src_shape[0], : src_shape[1]])


def run_patches(padded, patch_info, win, run_step, batch_size):
    """Per-patch network outputs [n,h,w,C] for every row of patch_info, in patch_info order.
    Multi-GPU: rank r runs the contiguous shard `shard_range(n, r, world)`; shards are padded to equal
    length and exchanged with one all_gather (NCCL on device tensors, gloo in the CPU tests)."""
    from ..dist import dist_info, shard_range

    n = patch_info.shape[0]
    dist, rank, world = dist_info()
    lo, hi = shard_range(n, rank, world)
    outs = []
    for b0 in range(lo, hi, batch_size):
        pi = patch_info[b0 : min(b0 + batch_size, hi)]
        batch = np.stack([padded[y : y + win, x : x + win] for y, x, _, _ in pi])
        outs.append(np.asarray(run_step(batch)))
    if world == 1:
        return np.concatenate(outs, axis=0)
    import torch
    probe = outs[0] if outs else np.asarray(run_step(np.stack([padded[:win, :win]])))  # shape of one output
    per = -(-n // world)
    mine = np.zeros((per,) + probe.shape[1:], dtype=np.float32)
    if outs:
        cat = np.concatenate(outs, axis=0)
        mine[: cat.shape[0]] = cat
    backend = dist.get_backend()
    t = torch.from_numpy(mine)
    t = t.cuda() if backend == "nccl" else t
    full = torch.empty((world * per,) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
    dist.all_gather_into_tensor(full, t)
    full = full.cpu().numpy()
    parts = []
    for r in range(world):
        l, h = shard_range(n, r, world)
        parts.append(full[r * per : r * per + (h - l)])
    return np.concatenate(parts, axis=0)


def _overlay(image, inst_dict, draw_dot=False, type_colour=None, line_thickness=2):
    """Contours (and optional centroid dots) over the image -- the role of reference
    misc/viz_utils.py:94-125; per-instance colours are seeded instead of the reference's shuffled HSV."""
    import cv2
    overlay = np.copy(image)
    rng = np.random.default_rng(0)
    for inst_id, info in inst_dict.items():
        if "type" in info and type_colour is not None and info["type"] in type_colour:
            colour = tuple(int(c) for c in type_colour[info["type"]][1])
        else:
            colour = tuple(int(c) for c in rng.integers(64, 256, 3))
        cv2.drawContours(overlay, [np.asarray(info["contour"], dtype=np.int32)], -1, colour, line_thickness)
        if draw_dot:
            overlay = cv2.circle(overlay, tuple(int(v) for v in info["centroid"]), 3, (255, 0, 0), -1)
    return overlay


def _to_qupath(file_path, nuc_pos_list, nuc_type_list, type_info_dict):
    """QuPath v0.2.3 TSV (reference convert_format.py:19-50)."""
    with open(file_path, "w") as fptr:
        fptr.write("x\ty\tclass\tname\tcolor\n")
        for pos, typ in zip(np.asarray(nuc_pos_list), np.asarray(nuc_type_list)):
            name, rgb = type_info_dict[typ][0], type_info_dict[typ][1]
            colour = (int(rgb[0]) << 16) + (int(rgb[1]) << 8) + int(rgb[2])
            fptr.write("{x}\t{y}\t{c}\t{n}\t{col}\n".format(x=pos[0], y=pos[1], c="", n=name, col=colour))


# Device bytes per image pixel of a tile group (hvn_infer_tiles_dev plus the caller's buffers): packed image 3, map 16,
# instance map 4, slot-order copies of both when sizes are mixed 20, padded instance table and contour counts
# 84 / 6 = 14 (each image's table holds min(rows_cap, H*W/6 + 8) rows, whatever the other sizes in the group), packed
# table and points ~2, post-processing workspace ~95 -- about 155, rounded up.  Per file on top: the 8 extra padded
# table rows (672 B), the default packed-table and point buffers of a small image (16 rows, 4096 points: 33 KB) and
# its slot entry.
DEVICE_BYTES_PER_PX = 192
DEVICE_BYTES_PER_FILE = 40 << 10
# With save_features: the prediction map the group keeps on the device for np_prob_mean (16) and the feature rows
# (18 x 8 B per table row, at most one row per 64 px by default: ~2.3).
FEATURE_BYTES_PER_PX = 20
_END = object()


def _padded_shape(h, w, win, step):
    """Shape of the reflect-padded image `_prepare_patching` builds for an h x w image."""
    last = lambda length: int((math.ceil((length - step) / step) + 1) * step)  # noqa: E731
    padt = (win - step) // 2
    return last(h) + win + padt, last(w) + win + padt, 3


def _file_cost(shape, win, step, features=False):
    """(RAM, device) bytes charged for one image of shape [H,W,3]: the reference's `sys.getsizeof(padded image) * 5`
    (infer/tile.py:271) and DEVICE_BYTES_PER_PX (+ FEATURE_BYTES_PER_PX with features) per pixel plus
    DEVICE_BYTES_PER_FILE."""
    ram = sys.getsizeof(np.empty(_padded_shape(shape[0], shape[1], win, step), dtype=np.uint8)) * 5
    per_px = DEVICE_BYTES_PER_PX + (FEATURE_BYTES_PER_PX if features else 0)
    return ram, per_px * int(shape[0]) * int(shape[1]) + DEVICE_BYTES_PER_FILE


def _groups(items, costs, budgets):
    """Cuts the stream `items` into groups, in order (reference infer/tile.py:236-290).  costs(item) -> (ram, device)
    bytes; budgets() -> (ram, device) bytes, read afresh for every group (device None: no device bound).  A group takes
    items while their summed costs stay within both budgets (the reference: `available_ram -= expected_usage; if
    available_ram < 0: break`).  It always takes at least one, so an item over the budget on its own is a group by
    itself -- the reference drops such a file without processing it."""
    it = iter(items)
    nxt = next(it, _END)
    while nxt is not _END:
        ram_budget, dev_budget = budgets()
        group, ram, dev = [], 0, 0
        while nxt is not _END:
            r, d = costs(nxt)
            if group and (ram + r > ram_budget or (dev_budget is not None and dev + d > dev_budget)):
                break
            group.append(nxt)
            ram, dev = ram + r, dev + d
            nxt = next(it, _END)
        yield group


def _rm_n_mkdir(path):
    if os.path.isdir(path):
        shutil.rmtree(path)
    os.makedirs(path)


class InferManager(base.InferManager):
    """Run inference on tiles."""

    def infer_image(self, img, all_ranks=False):
        """RGB uint8 [H,W,3] -> (pred_map [H,W,C] float32, pred_inst int32 [H,W], inst_info_dict).

        Device path (a manager built by `InferManager(**method_args)`): reflect padding, patch extraction,
        stitching, cropping, `process` and the contours all run in libhvn (`hvn_infer_tile`); only the image
        goes up and the maps / instance table / contour points come back.  With torch.distributed initialised
        on NCCL (one process per GPU) each rank runs its contiguous slice of the patch grid into a zeroed
        device map and the maps are summed onto rank 0 with one NCCL reduce (disjoint supports: x + 0 is exact); the
        single whole-map post-processing -- its min/max normalisations are global (SURVEY.md fact 6), so it cannot be
        sharded bit-exactly -- then runs ONCE, on rank 0; the other ranks return (None, None, None).  `all_ranks=True`
        all_reduces instead and post-processes everywhere (every rank gets the result; used by the 2-GPU parity test).
        Host path (fake `run_step` in the CPU tests, gloo): `run_patches` + `_stitch`."""
        from ..dist import dist_info, shard_range
        from ..models.hovernet.post_proc import table_to_dict

        dist, rank, world = dist_info()
        win = int(self.patch_input_shape)
        feats = getattr(self, "save_features", False)
        if getattr(self, "device_tile_path", False) and (world == 1 or dist.get_backend() == "nccl"):
            ctx = self.net.ctx
            if world == 1:
                if feats:
                    return self.infer_images([img])[0]
                pred_map, pred_inst, table, offs, pts = ctx.infer_tile(img, win, self.batch_size)
                return np.squeeze(pred_map), pred_inst, table_to_dict(table, offs, pts, self.nr_types)
            import torch
            H, W = img.shape[:2]
            rows, cols = ctx.tile_grid(H, W, win)
            lo, hi = shard_range(rows * cols, dist.get_rank(), world)
            d_img = torch.from_numpy(np.ascontiguousarray(img)).cuda()
            d_pred = torch.zeros((H, W, ctx.out_shape(win, win)[2]), dtype=torch.float32, device="cuda")
            torch.cuda.synchronize()  # torch's stream -> the library's stream
            ctx.tile_predict_dev(d_img.data_ptr(), H, W, win, lo, hi, self.batch_size, d_pred.data_ptr())
            ctx.sync()
            if all_ranks:
                dist.all_reduce(d_pred)
            else:
                dist.reduce(d_pred, dst=0)
                if rank != 0:
                    return None, None, None
            # whole-map post-processing + contours on the reduced map where it already lives: no 268 MB host round trip
            pred_inst, inst_info_dict = self._post_process_on_device(ctx, d_pred, H, W, d_img if feats else None)
            return np.squeeze(d_pred.cpu().numpy()), pred_inst, inst_info_dict
        else:
            src_shape = img.shape
            padded, patch_info, _ = _prepare_patching(img, self.patch_input_shape, self.patch_output_shape, True)
            outs = run_patches(padded, patch_info, self.patch_input_shape, self.run_step, self.batch_size)
            pred_map = _stitch(patch_info, outs, src_shape)
        if feats:
            from ..models.hovernet.post_proc import process_features
            pred_inst, inst_info_dict = process_features(pred_map, nr_types=self.nr_types, image=img)
            return np.squeeze(pred_map), pred_inst, inst_info_dict
        pred_inst, inst_info_dict = self.post_proc_func(pred_map, nr_types=self.nr_types, return_centroids=True)
        return np.squeeze(pred_map), pred_inst, inst_info_dict

    def infer_images(self, imgs, all_ranks=False):
        """A group of RGB uint8 images [H_i,W_i,3] -> one (pred_map, pred_inst, inst_info_dict) per image, each equal
        to `infer_image` on that image alone.

        Device path, one GPU: the patches of all images run as one stream of `batch_size` batches, and equal-size
        images are post-processed together (`hvn_infer_tiles`).  On several ranks (NCCL) each rank runs its contiguous
        slice of the group's combined patch list into a zeroed packed map, one NCCL reduce brings the maps to rank 0,
        and rank 0 post-processes each image (the other ranks get (None, None, None) per image; `all_ranks=True`
        all_reduces and post-processes everywhere).  Host path: `infer_image` per image."""
        from ..dist import dist_info, shard_range
        from ..models.hovernet.post_proc import table_to_dict

        dist, rank, world = dist_info()
        win = int(self.patch_input_shape)
        if not (getattr(self, "device_tile_path", False) and (world == 1 or dist.get_backend() == "nccl")):
            return [self.infer_image(img, all_ranks=all_ranks) for img in imgs]
        ctx = self.net.ctx
        feats = getattr(self, "save_features", False)
        if world == 1:
            return [(np.squeeze(r[0]), r[1], table_to_dict(r[2], r[3], r[4], self.nr_types, r[5] if feats else None))
                    for r in ctx.infer_tiles(imgs, win, self.batch_size, features=feats)]
        import torch
        C = ctx.out_shape(win, win)[2]
        grids = [ctx.tile_grid(img.shape[0], img.shape[1], win) for img in imgs]
        cells = np.cumsum([0] + [r * c for r, c in grids])
        px = np.cumsum([0] + [img.shape[0] * img.shape[1] for img in imgs])
        lo, hi = shard_range(int(cells[-1]), dist.get_rank(), world)
        d_pred = torch.zeros((int(px[-1]) * C,), dtype=torch.float32, device="cuda")
        mine = [i for i in range(len(imgs)) if cells[i] < hi and cells[i + 1] > lo]
        d_imgs = {i: torch.from_numpy(np.ascontiguousarray(imgs[i])).cuda() for i in mine}
        torch.cuda.synchronize()  # torch's stream -> the library's stream
        for i in mine:
            H, W = imgs[i].shape[:2]
            ctx.tile_predict_dev(d_imgs[i].data_ptr(), H, W, win, max(lo, int(cells[i])) - int(cells[i]),
                                 min(hi, int(cells[i + 1])) - int(cells[i]), self.batch_size,
                                 d_pred[int(px[i]) * C:].data_ptr())
        ctx.sync()
        if all_ranks:
            dist.all_reduce(d_pred)
        else:
            dist.reduce(d_pred, dst=0)
            if rank != 0:
                return [(None, None, None) for _ in imgs]
        out = []
        for i, img in enumerate(imgs):
            H, W = img.shape[:2]
            m = d_pred[int(px[i]) * C:int(px[i + 1]) * C].view(H, W, C)
            d_img = None
            if feats:
                d_img = d_imgs[i] if i in d_imgs else torch.from_numpy(np.ascontiguousarray(img)).cuda()
            pred_inst, inst_info_dict = self._post_process_on_device(ctx, m, H, W, d_img)
            out.append((np.squeeze(m.cpu().numpy()), pred_inst, inst_info_dict))
        return out

    def _post_process_on_device(self, ctx, d_pred, H, W, d_img=None):
        """`process` (post_proc.py:94-186) on a device-resident map [H,W,C]: hvn_postproc_dev + hvn_contours_dev, then
        only the instance map, the table rows and the contour points come back.  Same kernels as `post_proc.process`,
        hence the same result.  With d_img (the image [H,W,3] u8 on the device) the instances are also measured there
        (hvn_inst_features_dev)."""
        import torch
        from ..models.hovernet.post_proc import table_to_dict
        C = int(d_pred.shape[-1])
        max_rows, cap = max(16, H * W // 64), max(4096, H * W // 16)
        for _attempt in range(4):  # at most: grow the table once, then the point buffer once
            d_inst = torch.empty((H, W), dtype=torch.int32, device=d_pred.device)
            d_tab = torch.zeros((max_rows, 10), dtype=torch.int64, device=d_pred.device)
            d_nr = torch.zeros((1,), dtype=torch.int32, device=d_pred.device)
            d_offs = torch.zeros((max_rows + 1,), dtype=torch.int32, device=d_pred.device)
            d_pts = torch.empty((cap, 2), dtype=torch.int32, device=d_pred.device)
            torch.cuda.synchronize()  # torch's stream -> the library's stream
            ctx.postproc_dev(d_pred.data_ptr(), 1, H, W, C, self.nr_types, d_inst.data_ptr(), d_tab.data_ptr(), max_rows,
                             d_nr.data_ptr())
            ctx.contours_dev(d_inst.data_ptr(), d_tab.data_ptr(), d_nr.data_ptr(), 1, H, W, max_rows, d_pts.data_ptr(), cap,
                             d_offs.data_ptr())
            ctx.sync()
            n = int(d_nr.item())
            if n > max_rows:
                max_rows = n
                continue
            total = int(d_offs[max_rows].item())
            if total > cap:
                cap = total
                continue
            table = d_tab[:n].cpu().numpy()
            feats = None
            if d_img is not None:
                from .. import _lib
                d_ro = torch.tensor([0, n], dtype=torch.int32, device=d_pred.device)
                d_feats = torch.empty((max(1, n), _lib.FEAT_LEN), dtype=torch.float64, device=d_pred.device)
                torch.cuda.synchronize()
                ctx.inst_features_dev(1, [[H, W]], d_inst.data_ptr(), d_img.data_ptr(), d_pred.data_ptr(), C,
                                      d_tab.data_ptr(), d_ro.data_ptr(), n, d_pts.data_ptr(), d_offs.data_ptr(),
                                      d_feats.data_ptr())
                ctx.sync()
                feats = d_feats[:n].cpu().numpy()
            info = table_to_dict(table, d_offs.cpu().numpy(), d_pts[:total].cpu().numpy(), self.nr_types, feats)
            return d_inst.cpu().numpy(), info
        raise RuntimeError("tile post-processing: capacity retries exhausted")

    def process_file_list(self, run_args):
        """Process every image tile under run_args['input_dir'] (reference infer/tile.py:150-388), in groups of files
        (see the module docstring).  On several ranks every file is a group of its own: the ranks must form the same
        groups, and their free memory differs."""
        import cv2

        self.save_qupath = False
        self.save_raw_map = False
        self.save_features = False
        self.draw_dot = False
        self.mem_usage = 0.1
        self.batch_size = 32
        for variable, value in run_args.items():
            self.__setattr__(variable, value)
        assert self.mem_usage < 1.0 and self.mem_usage > 0.0
        patterning = lambda x: re.sub("([\\[\\]])", "[\\1]", x)  # noqa: E731
        file_path_list = glob.glob(patterning("%s/*" % self.input_dir))
        file_path_list.sort()  # ensure same order
        assert len(file_path_list) > 0, "Not Detected Any Files From Path"
        from ..dist import dist_info
        dist, rank, world = dist_info()
        multi = world > 1
        if rank == 0:  # every rank computes (the patch grid of each image is sharded); rank 0 alone writes
            for sub in ("json", "mat", "overlay"):
                _rm_n_mkdir(self.output_dir + "/%s/" % sub)
            if self.save_qupath:
                _rm_n_mkdir(self.output_dir + "/qupath/")
        if multi:
            dist.barrier()

        win, step = int(self.patch_input_shape), int(self.patch_output_shape)
        overlap = getattr(self, "device_tile_path", False) and not multi
        ctx = self.net.ctx if overlap else None

        def read(file_path):
            img = cv2.imread(file_path)
            if img is None:
                raise IOError("cannot read image %s" % file_path)
            return file_path, cv2.cvtColor(img, cv2.COLOR_BGR2RGB)

        def budgets():
            if multi:
                return -1, None
            import psutil
            ram = int(psutil.virtual_memory().available * self.mem_usage)
            # half of the free device memory: the other half stays for the network's activation plans (a new batch
            # tail builds one, up to ~18 GB for 32 original-mode patches) and the patch batches
            return ram, (ctx.mem_get_info()[0] // 2 if ctx is not None else None)

        groups = _groups((read(p) for p in file_path_list),
                         lambda f: _file_cost(f[1].shape, win, step, self.save_features), budgets)
        if not overlap:
            for files in groups:
                results = self.infer_images([img for _, img in files])
                if rank == 0:
                    self._write_files(files, results)
            return
        # one GPU: while group g runs on the device, group g-1's files are written and group g+1's files are read
        from ..models.hovernet.post_proc import table_to_dict
        files = next(groups, None)
        done = None  # (files, results) of the group whose outputs are still to be written
        while files is not None:
            job = ctx.infer_tiles_begin([img for _, img in files], win, self.batch_size, want_pred=self.save_raw_map,
                                        features=self.save_features)
            if done is not None:
                self._write_files(*done)
            upcoming = next(groups, None)
            results = [(None if r[0] is None else np.squeeze(r[0]), r[1],
                        table_to_dict(r[2], r[3], r[4], self.nr_types, r[5] if self.save_features else None))
                       for r in job.result()]
            done = (files, results)
            files = upcoming
        if done is not None:
            self._write_files(*done)
        return

    def _write_files(self, files, results):
        """The outputs of one group, file after file: `.mat`, overlay, QuPath TSV and JSON (reference
        infer/tile.py:326-369); with `save_features` also the `.mat`'s feature table."""
        import cv2
        import scipy.io as sio

        from .. import _lib

        for (file_path, img), (pred_map, pred_inst, inst_info_dict) in zip(files, results):
            img_name = pathlib.Path(file_path).stem
            nuc_val_list = list(inst_info_dict.values())
            nuc_uid_list = np.array(list(inst_info_dict.keys()))[:, None]  # singleton to make matlab happy
            nuc_type_list = np.array([v["type"] for v in nuc_val_list])[:, None]
            nuc_coms_list = np.array([v["centroid"] for v in nuc_val_list])
            mat_dict = {"inst_map": pred_inst, "inst_uid": nuc_uid_list, "inst_type": nuc_type_list,
                        "inst_centroid": nuc_coms_list}
            if self.nr_types is None:  # matlab does not have None type array
                mat_dict.pop("inst_type", None)
            if self.save_raw_map:
                mat_dict["raw_map"] = pred_map
            if getattr(self, "save_features", False):
                mat_dict["inst_features"] = np.array([[v["features"].get(k, np.nan) for k in _lib.FEATURE_NAMES]
                                                      for v in nuc_val_list], dtype=np.float64).reshape(-1, _lib.FEAT_LEN)
                mat_dict["inst_feature_names"] = np.array(_lib.FEATURE_NAMES, dtype=object)
            sio.savemat("%s/mat/%s.mat" % (self.output_dir, img_name), mat_dict)

            overlaid = _overlay(img, inst_info_dict, draw_dot=self.draw_dot,
                                type_colour=self.type_info_dict if self.nr_types is not None else None)
            cv2.imwrite("%s/overlay/%s.png" % (self.output_dir, img_name), cv2.cvtColor(overlaid, cv2.COLOR_RGB2BGR))
            if self.save_qupath:
                _to_qupath("%s/qupath/%s.tsv" % (self.output_dir, img_name), nuc_coms_list,
                           np.array([v["type"] for v in nuc_val_list]), self.type_info_dict)
            self._save_json("%s/json/%s.json" % (self.output_dir, img_name), inst_info_dict, None)
