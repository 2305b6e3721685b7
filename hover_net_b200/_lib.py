"""ctypes binding of libhvn.so (include/hvn.h).  There is no CPU fallback: if the CUDA library is
missing or no sm_90 device is present, every entry point raises."""
import ctypes
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libhvn.so")
ROW_LEN = 10
# hvn_targets flag bits (include/hvn.h HVN_TG_*): the maps the reference's gen_instance_hv_map raises ValueError on
TG_NO_BACKGROUND, TG_NO_BACKGROUND_CROP, TG_EMPTY_BOX = 1, 2, 4
# columns of hvn_inst_features (include/hvn.h HVN_FEAT_*), in order
FEATURE_NAMES = ("area", "contour_area", "perimeter", "convex_area", "solidity", "circularity", "major_axis_length",
                 "minor_axis_length", "eccentricity", "orientation", "feret_max", "mean_r", "mean_g", "mean_b", "std_r",
                 "std_g", "std_b", "np_prob_mean")
FEAT_LEN = len(FEATURE_NAMES)
_lib = None


class HvnError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("libhvn error %d: %s" % (code, msg))
        self.code = code


# The C ABI of include/hvn.h as ctypes sees it: name -> (restype, argtypes).  Every pointer is c_void_p, `const char *`
# is c_char_p; lib() applies the table when the library loads.
_P, _S, _I, _I64, _SZ = ctypes.c_void_p, ctypes.c_char_p, ctypes.c_int, ctypes.c_int64, ctypes.c_size_t
_VALID = [_P, _P, _P, _P, _I, _I, _I, _P, _P, _P]
_TILES_ARGS = [_P, _I, _P, _P, _I, _I, _P, _P, _P, _I64, _P, _P, _I64, _P]
_FEAT_ARGS = [_P, _I, _P, _P, _P, _P, _I, _P, _P, _I64, _P, _P, _P]
PROTOTYPES = {
    "hvn_abi_version": (_I, []),
    "hvn_last_error": (_S, []),
    "hvn_create": (_I, [_I, _S, _I, _P]),
    "hvn_destroy": (None, [_P]),
    "hvn_num_params": (_I, [_P]),
    "hvn_param_info": (_I, [_P, _I, _P, _P, _P]),
    "hvn_load_param": (_I, [_P, _S, _P, _I, _P]),
    "hvn_finalize_weights": (_I, [_P]),
    "hvn_set_option": (_I, [_P, _S, _I64]),
    "hvn_debug_log": (_S, [_P]),
    "hvn_get_counter": (_I64, [_P, _S]),
    "hvn_out_shape": (_I, [_P, _I, _I, _P, _P, _P]),
    "hvn_forward": (_I, [_P, _P, _I, _I, _I, _P]),
    "hvn_forward_dev": (_I, [_P, _P, _I, _I, _I, _P]),
    "hvn_create_postproc": (_I, [_I, _P]),
    "hvn_postproc": (_I, [_P, _P, _I, _I, _I, _I, _I, _P, _P, _I, _P]),
    "hvn_postproc_dev": (_I, [_P, _P, _I, _I, _I, _I, _I, _P, _P, _I, _P]),
    "hvn_contours_dev": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _P, _I64, _P]),
    "hvn_postproc_contours": (_I, [_P, _P, _I, _I, _I, _I, _I, _P, _P, _I, _P, _P, _I64, _P]),
    "hvn_forward_postproc": (_I, [_P, _P, _I, _I, _I, _P, _P, _P, _I, _P]),
    "hvn_forward_postproc_dev": (_I, [_P, _P, _I, _I, _I, _P, _P, _P, _I, _P]),
    "hvn_tile_grid": (_I, [_P, _I, _I, _I, _P, _P]),
    "hvn_tile_predict_dev": (_I, [_P, _P, _I, _I, _I, _I, _I, _I, _P]),
    "hvn_infer_tile": (_I, [_P, _P, _I, _I, _I, _I, _P, _P, _P, _I, _P, _P, _I64, _P]),
    "hvn_infer_tiles": (_I, _TILES_ARGS),
    "hvn_infer_tiles_dev": (_I, _TILES_ARGS),
    "hvn_pack_tables_dev": (_I, [_P, _P, _P, _I, _I, _P, _I64, _P]),
    "hvn_get_stream": (_I, [_P, _P]),
    "hvn_inst_pairs": (_I, [_P, _P, _P, _I, _I, _I, _P, _I64, _P]),
    "hvn_inst_pairs_dev": (_I, [_P, _P, _P, _I, _I, _I, _P, _I64, _P]),
    "hvn_targets": (_I, [_P, _P, _I, _I, _I, _I, _I, _P, _P]),
    "hvn_targets_dev": (_I, [_P, _P, _I, _I, _I, _I, _I, _P, _P]),
    "hvn_valid": (_I, _VALID),
    "hvn_valid_dev": (_I, _VALID),
    "hvn_valid_loss": (_I, _VALID + [_P, _P]),
    "hvn_valid_loss_dev": (_I, _VALID + [_P, _P]),
    "hvn_inst_features": (_I, _FEAT_ARGS),
    "hvn_inst_features_dev": (_I, _FEAT_ARGS),
    "hvn_malloc": (_I, [_P, _SZ, _P]),
    "hvn_free": (_I, [_P, _P]),
    "hvn_malloc_host": (_I, [_P, _SZ, _P]),
    "hvn_free_host": (_I, [_P, _P]),
    "hvn_memcpy_h2d": (_I, [_P, _P, _P, _SZ]),
    "hvn_memcpy_d2h": (_I, [_P, _P, _P, _SZ]),
    "hvn_sync": (_I, [_P]),
    "hvn_mem_info": (_I, [_P, _P, _P]),
    "hvn_timer_start": (_I, [_P]),
    "hvn_timer_stop": (_I, [_P, _P]),
    "hvn_stage_ms": (_I, [_P, _S, _P]),
}


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise HvnError(-2, "libhvn.so is not built (run `python -c 'import __graft_entry__ as g; g.build()'`); "
                               "this package has no CPU fallback")
        L = ctypes.CDLL(LIB_PATH)
        for name, (restype, argtypes) in PROTOTYPES.items():
            f = getattr(L, name)
            f.restype, f.argtypes = restype, argtypes
        _lib = L
    return _lib


def check(rc):
    if rc != 0:
        raise HvnError(rc, lib().hvn_last_error().decode("utf-8", "replace"))


def _retry_capacity(what, attempt):
    """Runs attempt() -> (rc, result) until rc is not HVN_ERR_CAPACITY (-4), at most 4 times, and returns result; any
    other failure raises.  On -4, attempt has taken the exact sizes the call reported for its next run."""
    for _attempt in range(4):
        rc, result = attempt()
        if rc != -4:
            check(rc)
            return result
    raise HvnError(-4, "%s: capacity retries exhausted" % what)


def _ptr(a):
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        return a.ctypes.data_as(ctypes.c_void_p)
    return ctypes.c_void_p(int(a))  # raw address (device pointer or pinned host)


PRECISIONS = {"highest": 0, "high": 1}


def precision_code(precision):
    """"highest" -> 0, "high" -> 1 (libhvn option "precision"); anything else is a ValueError, raised before any
    device is touched."""
    if precision not in PRECISIONS:
        raise ValueError("precision must be one of %s, got %r" % (sorted(PRECISIONS), precision))
    return PRECISIONS[precision]


def tta_code(tta):
    """True -> 1, False -> 0 (libhvn option "tta"); anything but a bool is a ValueError, raised before any device is
    touched."""
    if not isinstance(tta, bool):
        raise ValueError("tta must be True or False, got %r" % (tta,))
    return int(tta)


def _as_ids(a):
    """Instance map as C-contiguous int32; ids that int32 cannot hold are an error, never wrapped."""
    a = np.asarray(a)
    if a.dtype == np.int32:
        return np.ascontiguousarray(a)
    b = np.ascontiguousarray(a, dtype=np.int32)
    if not np.array_equal(b, a):
        raise ValueError("instance ids must be integers that fit in int32")
    return b


def pack_images(imgs):
    """RGB images [H_i,W_i,3] -> (uint8 [sum H_i*W_i*3] back to back in input order, shapes int32 [n,2] = (H_i, W_i)):
    the input of hvn_infer_tiles."""
    arrs = [np.ascontiguousarray(a, dtype=np.uint8) for a in imgs]
    for a in arrs:
        if a.ndim != 3 or a.shape[2] != 3:
            raise ValueError("tile images must be RGB [H,W,3], got %s" % (a.shape,))
    shapes = np.array([a.shape[:2] for a in arrs], dtype=np.int32).reshape(-1, 2)
    packed = np.concatenate([a.reshape(-1) for a in arrs]) if arrs else np.zeros((0,), np.uint8)
    return packed, shapes


def tiles_sizes(shapes):
    """Default (rows_cap, pts_cap) of a tile group: hvn_infer_tile's per-image defaults, summed."""
    px = [int(h) * int(w) for h, w in np.asarray(shapes).reshape(-1, 2)]
    return sum(max(16, p // 64) for p in px), sum(max(4096, p // 16) for p in px)


def split_tiles(shapes, inst, table, row_offs, pred=None, pts=None, pt_offs=None, feats=None):
    """Packed outputs of hvn_infer_tiles -> one (pred [H,W,C] or None, inst [H,W], table [k,10], offs [k+1], pts [m,2]
    or None) per image, the tuple Context.infer_tile returns: offs index the image's own points.  With feats (the
    group's hvn_inst_features rows [rows,FEAT_LEN]) each tuple gains the image's rows of it."""
    out = []
    p0 = 0
    C = None if pred is None else pred.size // max(1, int(sum(int(h) * int(w) for h, w in shapes)))
    for i, (h, w) in enumerate(np.asarray(shapes).reshape(-1, 2)):
        h, w = int(h), int(w)
        r0, r1 = int(row_offs[i]), int(row_offs[i + 1])
        pm = None if pred is None else pred[p0 * C:(p0 + h * w) * C].reshape(h, w, C)
        im = inst[p0:p0 + h * w].reshape(h, w)
        offs = pt = None
        if pt_offs is not None:
            offs = np.asarray(pt_offs[r0:r1 + 1], dtype=np.int64) - int(pt_offs[r0])
            pt = pts[int(pt_offs[r0]):int(pt_offs[r1])]
        out.append((pm, im, table[r0:r1], offs, pt) + (() if feats is None else (feats[r0:r1],)))
        p0 += h * w
    return out


class TilesJob:
    """A tile group enqueued with hvn_infer_tiles_dev (Context.infer_tiles_begin).  result() synchronises and returns
    what Context.infer_tiles returns.  A capacity failure reruns the group through Context.infer_tiles with the sizes the
    offsets report; a range failure reruns it there too, which raises act_shift.  With features, result() measures
    every instance (hvn_inst_features_dev) on the group's device image, instance and prediction maps before they are
    freed; the prediction map is kept on the device for that even when it is not wanted back.  Such a group is rerun
    as another TilesJob (the maps are measured on the device there too): with the reported sizes after a capacity
    failure, with act_shift raised by 6 after a range failure, as Context._retry_range does."""

    MAX_RERUNS = 9  # two capacity growths and six act_shift steps, and one to spare

    def __init__(self, ctx, imgs, patch_in, batch, want_pred, contours, features=False, rows_cap=None, pts_cap=None,
                 reruns=0):
        if features and not contours:
            raise ValueError("instance features need the contours")
        self.ctx, self.imgs, self.patch_in, self.batch = ctx, imgs, patch_in, batch
        self.want_pred, self.contours, self.features, self.reruns = want_pred, contours, features, reruns
        self.packed, self.shapes = pack_images(imgs)
        n = self.shapes.shape[0]
        px = int(self.packed.size // 3)
        self.oc = ctx.out_shape(patch_in, patch_in)[2]
        r0, p0 = tiles_sizes(self.shapes)
        self.rows_cap = r0 if rows_cap is None else int(rows_cap)
        self.pts_cap = p0 if pts_cap is None else int(pts_cap)
        sizes = {"img": px * 3, "pred": px * self.oc * 4 if want_pred or features else 0, "inst": px * 4,
                 "table": self.rows_cap * ROW_LEN * 8, "ro": (n + 1) * 4,
                 "po": (self.rows_cap + 1) * 4 if contours else 0, "pts": self.pts_cap * 8 if contours else 0}
        self.d = {k: (ctx.malloc(b) if b else None) for k, b in sizes.items()}
        try:
            ctx.h2d(self.d["img"], self.packed, self.packed.nbytes)
            check(lib().hvn_infer_tiles_dev(ctx._h, n, _ptr(self.d["img"]), _ptr(self.shapes), int(patch_in), int(batch),
                                            _ptr(self.d["pred"]), _ptr(self.d["inst"]), _ptr(self.d["table"]),
                                            int(self.rows_cap), _ptr(self.d["ro"]), _ptr(self.d["pts"]),
                                            int(self.pts_cap if contours else 0), _ptr(self.d["po"])))
        except Exception:
            self._free()
            raise

    def _free(self):
        for k, p in self.d.items():
            if p:
                self.ctx.free(p)
        self.d = {}

    def result(self):
        ctx, n = self.ctx, self.shapes.shape[0]
        try:
            try:
                ctx.sync()
            except HvnError as e:
                if e.code != -6:
                    raise
                return self._rerun(range_failed=True)
            ro = np.zeros((n + 1,), dtype=np.int32)
            ctx.d2h(ro, self.d["ro"], ro.nbytes)
            rows = int(ro[-1])
            po = None
            if self.contours:
                po = np.zeros((self.rows_cap + 1,), dtype=np.int32)
                if rows <= self.rows_cap:
                    ctx.d2h(po, self.d["po"], po.nbytes)
            if rows > self.rows_cap:
                return self._rerun(rows_cap=rows)  # the points are sized on the rerun's own retry if need be
            if po is not None and int(po[rows]) > self.pts_cap:
                return self._rerun(rows_cap=self.rows_cap, pts_cap=int(po[rows]))
            px = int(self.packed.size // 3)
            inst = np.empty((px,), dtype=np.int32)
            ctx.d2h(inst, self.d["inst"], inst.nbytes)
            table = np.empty((rows, ROW_LEN), dtype=np.int64)
            if rows:
                ctx.d2h(table, self.d["table"], table.nbytes)
            pred = pts = None
            if self.want_pred:
                pred = np.empty((px * self.oc,), dtype=np.float32)
                ctx.d2h(pred, self.d["pred"], pred.nbytes)
            if self.contours:
                pts = np.empty((int(po[rows]), 2), dtype=np.int32)
                if pts.size:
                    ctx.d2h(pts, self.d["pts"], pts.nbytes)
                po = po[: rows + 1]
            feats = None
            if self.features:
                feats = np.empty((rows, FEAT_LEN), dtype=np.float64)
                d_feats = ctx.malloc(max(1, feats.nbytes))
                try:
                    ctx.inst_features_dev(n, self.shapes, self.d["inst"], self.d["img"], self.d["pred"], self.oc,
                                          self.d["table"], self.d["ro"], rows, self.d["pts"], self.d["po"], d_feats)
                    if rows:
                        ctx.d2h(feats, d_feats, feats.nbytes)
                    ctx.sync()
                finally:
                    ctx.free(d_feats)
            ctx.sync()
            return split_tiles(self.shapes, inst, table, ro, pred, pts, po, feats)
        finally:
            self._free()

    def _rerun(self, rows_cap=None, pts_cap=None, range_failed=False):
        """The group again, with the exact sizes when a capacity check failed: through the synchronising host variant,
        or with features as another TilesJob."""
        self._free()
        if not self.features:
            return self.ctx.infer_tiles(self.imgs, self.patch_in, self.batch, want_pred=self.want_pred,
                                        contours=self.contours, rows_cap=rows_cap, pts_cap=pts_cap)
        if self.reruns >= self.MAX_RERUNS:
            raise HvnError(-4 if not range_failed else -6, "tile group with features: reruns exhausted")
        if range_failed:
            self.ctx.set_option("act_shift", self.ctx.counter("act_shift") + 6)
        return TilesJob(self.ctx, self.imgs, self.patch_in, self.batch, self.want_pred, self.contours, True,
                        rows_cap or self.rows_cap, pts_cap or self.pts_cap, self.reruns + 1).result()


class Context:
    """One libhvn context (one device, one stream).  precision: "highest" (default; fp16 hi + lo operands, three
    products per MAC) or "high" (hi only, one fp16 product per MAC -- TF32-class operand precision); model contexts
    only, set before any weights are finalised.  tta (an extension the reference lacks): True runs every patch as its
    eight dihedral views (4 rotations x optional mirror) and averages their maps, HV vectors mapped back, on the device
    before post-processing; square patches only; 8x the network work."""

    def __init__(self, device=0, mode=None, nr_types=None, precision="highest", tta=False):
        code = precision_code(precision)
        tta_on = tta_code(tta)
        self._h = ctypes.c_void_p()
        L = lib()
        if mode is None:
            check(L.hvn_create_postproc(int(device), ctypes.byref(self._h)))
        else:
            check(L.hvn_create(int(device), mode.encode(), int(nr_types or 0), ctypes.byref(self._h)))
            if code:
                self.set_option("precision", code)
            if tta_on:
                self.set_option("tta", tta_on)
        self.device = int(device)
        self.mode = mode
        self.nr_types = nr_types
        self.precision = precision
        self.tta = tta
        for kv in os.environ.get("HVN_OPTS", "").split(","):  # development knobs: HVN_OPTS="key=value,..."
            if "=" in kv and mode is not None:
                k, v = kv.split("=")
                self.set_option(k.strip(), int(v))

    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            lib().hvn_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- weights
    def param_specs(self):
        L = lib()
        out = []
        name = ctypes.c_char_p()
        ndim = ctypes.c_int()
        shape = (ctypes.c_int64 * 4)()
        for i in range(L.hvn_num_params(self._h)):
            check(L.hvn_param_info(self._h, i, ctypes.byref(name), ctypes.byref(ndim), shape))
            out.append((name.value.decode(), tuple(int(shape[j]) for j in range(ndim.value))))
        return out

    def load_param(self, name, array):
        a = np.ascontiguousarray(np.asarray(array), dtype=np.float32)
        shape = (ctypes.c_int64 * 4)(*(list(a.shape) + [0] * (4 - a.ndim)))
        check(lib().hvn_load_param(self._h, name.encode(), _ptr(a), a.ndim, shape))

    def finalize_weights(self):
        check(lib().hvn_finalize_weights(self._h))

    def set_option(self, key, value):
        check(lib().hvn_set_option(self._h, key.encode(), int(value)))

    def debug_log(self):
        return lib().hvn_debug_log(self._h).decode("utf-8", "replace")

    def counter(self, key):
        return int(lib().hvn_get_counter(self._h, key.encode()))

    def out_shape(self, h, w):
        oh, ow, oc = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
        check(lib().hvn_out_shape(self._h, int(h), int(w), ctypes.byref(oh), ctypes.byref(ow), ctypes.byref(oc)))
        return oh.value, ow.value, oc.value

    def _retry_range(self, call):
        """Runs call() -> rc.  HVN_ERR_RANGE (-6: an activation outside the fp16 hi+lo range) is answered by raising
        the exact power-of-two activation scale (option "act_shift", +6 per attempt) and running again -- the result
        is never a silently clamped map.  The shift is kept for later calls."""
        rc = call()
        tries = 0
        while rc == -6 and tries < 6:
            tries += 1
            self.set_option("act_shift", self.counter("act_shift") + 6)
            rc = call()
        return rc

    # ---- host-buffer entry points (what the reference-facing plugin calls)
    def forward(self, imgs_u8, out=None):
        x = np.ascontiguousarray(imgs_u8, dtype=np.uint8)
        B, H, W, C = x.shape
        assert C == 3
        oh, ow, oc = self.out_shape(H, W)
        if out is None:
            out = np.empty((B, oh, ow, oc), dtype=np.float32)
        check(self._retry_range(lambda: lib().hvn_forward(self._h, _ptr(x), B, H, W, _ptr(out))))
        return out

    def postproc(self, pred, nr_types=None, max_rows=None):
        p = np.ascontiguousarray(pred, dtype=np.float32)
        if p.ndim == 3:
            p = p[None]
        n, H, W, C = p.shape
        if max_rows is None:
            max_rows = max(16, H * W // 64)

        def attempt():
            nonlocal max_rows
            inst = np.empty((n, H, W), dtype=np.int32)
            table = np.zeros((n, max_rows, ROW_LEN), dtype=np.int64)
            nrows = np.zeros((n,), dtype=np.int32)
            rc = lib().hvn_postproc(self._h, _ptr(p), n, H, W, C, int(nr_types or 0), _ptr(inst), _ptr(table),
                                    int(max_rows), _ptr(nrows))
            if rc == -4:
                max_rows = int(nrows.max())
            return rc, (inst, table, nrows)
        return _retry_capacity("postproc", attempt)

    def postproc_contours(self, pred, nr_types=None, max_rows=None, pts_cap=None):
        """postproc + device contour tracing: (inst, table, nrows, offs [n*max_rows+1], pts [total,2])."""
        p = np.ascontiguousarray(pred, dtype=np.float32)
        if p.ndim == 3:
            p = p[None]
        n, H, W, C = p.shape
        if max_rows is None:
            max_rows = max(16, H * W // 64)
        if pts_cap is None:
            pts_cap = max(4096, n * H * W // 16)

        def attempt():  # a capacity failure grows the table once, then the point buffer once
            nonlocal max_rows, pts_cap
            inst = np.empty((n, H, W), dtype=np.int32)
            table = np.zeros((n, max_rows, ROW_LEN), dtype=np.int64)
            nrows = np.zeros((n,), dtype=np.int32)
            offs = np.zeros((n * max_rows + 1,), dtype=np.int32)
            pts = np.empty((pts_cap, 2), dtype=np.int32)
            rc = lib().hvn_postproc_contours(self._h, _ptr(p), n, H, W, C, int(nr_types or 0), _ptr(inst), _ptr(table),
                                             int(max_rows), _ptr(nrows), _ptr(pts), int(pts_cap), _ptr(offs))
            if rc == -4:
                if int(nrows.max()) > max_rows:
                    max_rows = int(nrows.max())
                else:
                    pts_cap = int(offs[-1])
            return rc, (inst, table, nrows, offs, pts[: int(offs[-1])])
        return _retry_capacity("postproc_contours", attempt)

    def contours_dev(self, d_inst, d_table, d_nrows, n, H, W, max_rows, d_pts, pts_cap, d_offs):
        check(lib().hvn_contours_dev(self._h, _ptr(d_inst), _ptr(d_table), _ptr(d_nrows), n, H, W, int(max_rows),
                                     _ptr(d_pts), int(pts_cap), _ptr(d_offs)))

    def inst_pairs(self, true, pred=None, cap=None):
        """Contingency table of instance maps true/pred [H,W] or [n,H,W] (ids >= 0, 0 = background; pred None = all
        zero).  Returns (rows [total,3] int64 (t, p, count), offs [n+1] int64): the rows of map m are
        rows[offs[m]:offs[m+1]], every (t, p) with t > 0 or p > 0 that occurs, sorted by (t, p)."""
        t = _as_ids(true)
        p = None if pred is None else _as_ids(pred)
        if t.ndim == 2:
            t = t[None]
            p = None if p is None else p[None]
        if p is not None and p.shape != t.shape:
            raise ValueError("true and pred shapes differ: %s vs %s" % (t.shape, p.shape))
        n, H, W = t.shape
        if cap is None:
            cap = max(1024, n * H * W // 64)

        def attempt():
            nonlocal cap
            rows = np.empty((cap, 3), dtype=np.int64)
            offs = np.zeros((n + 1,), dtype=np.int64)
            rc = lib().hvn_inst_pairs(self._h, _ptr(t), _ptr(p), n, H, W, _ptr(rows), int(cap), _ptr(offs))
            if rc == -4:
                cap = int(offs[-1])
            return rc, (rows[: int(offs[-1])], offs)
        rows, offs = _retry_capacity("inst_pairs", attempt)
        m = np.repeat(np.arange(n), np.diff(offs))
        return rows[np.lexsort((rows[:, 1], rows[:, 0], m))], offs

    def inst_pairs_dev(self, d_true, d_pred, n, H, W, d_pairs, cap, d_offs):
        """Device-pointer variant (d_pred may be None).  Returns False on HVN_ERR_CAPACITY (offs is valid on the
        device then: retry with cap >= offs[n]), True on success; raises on any other error."""
        rc = lib().hvn_inst_pairs_dev(self._h, _ptr(d_true), _ptr(d_pred), int(n), int(H), int(W), _ptr(d_pairs),
                                      int(cap), _ptr(d_offs))
        if rc == -4:
            return False
        check(rc)
        return True

    def targets(self, inst, crop_shape):
        """Full-size HV targets of instance maps inst [H,W] or [n,H,W] (the reference's gen_instance_hv_map):
        returns (hv float32 [n,H,W,2] (x, y), flags int32 [n] -- TG_* bits, the maps the reference rejects)."""
        a = _as_ids(inst)
        if a.ndim == 2:
            a = a[None]
        n, H, W = a.shape
        hv = np.empty((n, H, W, 2), dtype=np.float32)
        flags = np.zeros((n,), dtype=np.int32)
        check(lib().hvn_targets(self._h, _ptr(a), n, H, W, int(crop_shape[0]), int(crop_shape[1]), _ptr(hv), _ptr(flags)))
        return hv, flags

    def targets_dev(self, d_inst, n, H, W, crop_h, crop_w, d_hv, d_flags):
        check(lib().hvn_targets_dev(self._h, _ptr(d_inst), int(n), int(H), int(W), int(crop_h), int(crop_w), _ptr(d_hv),
                                    _ptr(d_flags)))

    # argument list of hvn_valid_loss*, for callers that set a function's argtypes themselves (as _TILES_ARGS)
    _VALID_LOSS_ARGS = PROTOTYPES["hvn_valid_loss"][1]

    def _valid_args(self, imgs_u8, inst, type_map):
        """The inputs of a validation batch as the C ABI takes them, and its zeroed counts, hv_sse and flags."""
        x = np.ascontiguousarray(imgs_u8, dtype=np.uint8)
        B, H, W, C = x.shape
        assert C == 3
        a = _as_ids(inst)
        t = None if type_map is None or not self.nr_types else _as_ids(type_map)
        if a.shape != (B, H, W) or (t is not None and t.shape != (B, H, W)):
            raise ValueError("inst / type maps must be [B,H,W] = %s" % ((B, H, W),))
        counts = np.zeros((3 + 2 * int(self.nr_types or 0),), dtype=np.int64)
        return x, a, t, counts, np.zeros((1,), dtype=np.float64), np.zeros((B,), dtype=np.int32)

    def valid(self, imgs_u8, inst, type_map=None):
        """One validation batch through forward, targets and counts on the device (model contexts).  imgs uint8
        [B,H,W,3], inst / type_map int32 [B,H,W] at the network input size.  Returns (counts int64 [3 + 2*nr_types]
        = correct, inter, total, then inter_k, total_k per type; hv_sse float; flags int32 [B])."""
        x, a, t, counts, sse, flags = self._valid_args(imgs_u8, inst, type_map)
        B, H, W, _ = x.shape
        check(self._retry_range(lambda: lib().hvn_valid(self._h, _ptr(x), _ptr(a), _ptr(t), B, H, W, _ptr(counts),
                                                        _ptr(sse), _ptr(flags))))
        return counts, float(sse[0]), flags

    def valid_dev(self, d_imgs, d_inst, d_type, B, H, W, d_counts, d_sse, d_flags):
        check(lib().hvn_valid_dev(self._h, _ptr(d_imgs), _ptr(d_inst), _ptr(d_type), int(B), int(H), int(W),
                                  _ptr(d_counts), _ptr(d_sse), _ptr(d_flags)))

    def valid_loss(self, imgs_u8, inst, type_map=None, want_probs=False):
        """`valid` plus the reference's training-loss sums on the same eval-mode forward (hvn_valid_loss).  Returns
        (counts, hv_sse, flags) as `valid` does, then sums float64 [10 + (1 + 3*nr_types if typed)] (layout in
        include/hvn.h; run_desc.loss_scalars turns them into the loss values) and, with want_probs, the probability
        map float32 [B,h,w,4+nr_types] = [np p0, np p1, hv x, hv y, tp p0..] (else None).  A type id outside
        0..nr_types-1 inside the output crop raises HvnError (HVN_ERR_INVALID)."""
        x, a, t, counts, sse, flags = self._valid_args(imgs_u8, inst, type_map)
        B, H, W, _ = x.shape
        nt = int(self.nr_types or 0)
        sums = np.zeros((10 + (1 + 3 * nt if nt else 0),), dtype=np.float64)
        probs = None
        if want_probs:
            oh, ow, _ = self.out_shape(H, W)
            probs = np.empty((B, oh, ow, 4 + nt), dtype=np.float32)
        check(self._retry_range(lambda: lib().hvn_valid_loss(self._h, _ptr(x), _ptr(a), _ptr(t), B, H, W, _ptr(counts),
                                                             _ptr(sse), _ptr(flags), _ptr(sums), _ptr(probs))))
        return counts, float(sse[0]), flags, sums, probs

    def valid_loss_dev(self, d_imgs, d_inst, d_type, B, H, W, d_counts, d_sse, d_flags, d_sums, d_probs=None):
        check(lib().hvn_valid_loss_dev(self._h, _ptr(d_imgs), _ptr(d_inst), _ptr(d_type), int(B), int(H), int(W),
                                       _ptr(d_counts), _ptr(d_sse), _ptr(d_flags), _ptr(d_sums), _ptr(d_probs)))

    def _features_packed(self, shapes, inst, img, pred, C, table, row_offs, pts, pt_offs):
        """hvn_inst_features on host arrays already in the packed layout; returns feats [n_rows,FEAT_LEN]."""
        sh = np.ascontiguousarray(shapes, dtype=np.int32).reshape(-1, 2)
        n_rows = int(row_offs[-1])
        feats = np.empty((n_rows, FEAT_LEN), dtype=np.float64)
        c = lambda a, t: None if a is None else np.ascontiguousarray(a, dtype=t)  # noqa: E731
        check(lib().hvn_inst_features(
            self._h, sh.shape[0], _ptr(sh), _ptr(c(inst, np.int32)), _ptr(c(img, np.uint8)), _ptr(c(pred, np.float32)),
            int(C), _ptr(c(table, np.int64)), _ptr(c(row_offs, np.int32)), n_rows, _ptr(c(pts, np.int32)),
            _ptr(c(pt_offs, np.int32)), _ptr(feats)))
        return feats

    def inst_features(self, inst, table, pts, pt_offs, row_offs=None, image=None, pred=None):
        """Per-instance measurements (hvn_inst_features; columns FEATURE_NAMES) of the rows of `table`.
        inst: one instance map [H,W] or a list of maps of any sizes; image / pred: None or the matching RGB uint8
        [H,W,3] (any other dtype is a ValueError) / prediction [H,W,C] maps (NP at channel C - 3; their columns are NaN when None); table [n,10];
        row_offs [n_maps+1] (default [0, n] for one map); the contour of row r at pts[pt_offs[r]:pt_offs[r+1]], (x, y)
        in map coordinates.  Returns float64 [n,FEAT_LEN]."""
        many = isinstance(inst, (list, tuple))
        maps = [_as_ids(m) for m in (inst if many else [inst])]
        imgs = None if image is None else [np.asarray(a) for a in (image if many else [image])]
        if imgs is not None and any(a.dtype != np.uint8 for a in imgs):
            raise ValueError("images must be uint8 RGB (the colour columns are statistics of 0..255 values), got %s"
                             % sorted(set(str(a.dtype) for a in imgs)))
        preds = None if pred is None else [np.asarray(a) for a in (pred if many else [pred])]
        for k, m in enumerate(maps):
            if m.ndim != 2 or (imgs is not None and imgs[k].shape != m.shape + (3,)) or \
                    (preds is not None and (preds[k].ndim != 3 or preds[k].shape[:2] != m.shape)):
                raise ValueError("map %d: inst [H,W], image [H,W,3] and pred [H,W,C] must agree" % k)
        C = preds[0].shape[2] if preds is not None else 0
        table = np.ascontiguousarray(table, dtype=np.int64).reshape(-1, ROW_LEN)
        if row_offs is None:
            if many and len(maps) != 1:
                raise ValueError("row_offs is needed with more than one map")
            row_offs = [0, table.shape[0]]
        row_offs = np.ascontiguousarray(row_offs, dtype=np.int32)
        n_rows = int(row_offs[-1])
        if n_rows != table.shape[0]:
            raise ValueError("row_offs[-1] = %d but the table has %d rows" % (n_rows, table.shape[0]))
        cat = lambda arrs: None if arrs is None else np.concatenate([a.reshape(-1) for a in arrs])  # noqa: E731
        shapes = np.array([m.shape for m in maps], dtype=np.int32)
        pts = np.asarray(pts).reshape(-1, 2) if pts is not None else np.zeros((0, 2), np.int32)
        pt_offs = np.asarray(pt_offs)[: n_rows + 1]
        if pt_offs.size != n_rows + 1 or not 0 <= int(pt_offs[0]) <= int(pt_offs[-1]) <= pts.shape[0]:
            raise ValueError("pt_offs needs n_rows + 1 entries with 0 <= pt_offs[0] <= pt_offs[n_rows] <= %d (the "
                             "points given)" % pts.shape[0])
        return self._features_packed(shapes, cat(maps), cat(imgs), cat(preds), C, table, row_offs, pts, pt_offs)

    def inst_features_dev(self, n_maps, shapes, d_inst, d_img, d_pred, C, d_table, d_row_offs, n_rows, d_pts, d_pt_offs,
                          d_feats):
        """hvn_inst_features_dev on device pointers (shapes: host int32 [n_maps,2]; d_img / d_pred may be None)."""
        sh = np.ascontiguousarray(shapes, dtype=np.int32)
        check(lib().hvn_inst_features_dev(self._h, int(n_maps), _ptr(sh), _ptr(d_inst), _ptr(d_img), _ptr(d_pred), int(C),
                                          _ptr(d_table), _ptr(d_row_offs), int(n_rows), _ptr(d_pts), _ptr(d_pt_offs),
                                          _ptr(d_feats)))

    def mem_get_info(self):
        """(free, total) device bytes of this context's device (hvn_mem_info)."""
        free, total = ctypes.c_size_t(), ctypes.c_size_t()
        check(lib().hvn_mem_info(self._h, ctypes.byref(free), ctypes.byref(total)))
        return int(free.value), int(total.value)

    def tile_grid(self, H, W, patch_in):
        r, c = ctypes.c_int(), ctypes.c_int()
        check(lib().hvn_tile_grid(self._h, int(H), int(W), int(patch_in), ctypes.byref(r), ctypes.byref(c)))
        return r.value, c.value

    def infer_tile(self, img_u8, patch_in, batch=0, want_pred=True, contours=True, max_rows=None, pts_cap=None):
        """One RGB image [H,W,3] through the device tile path (reflect pad, patches, network, stitch, crop,
        process, contours).  Returns (pred or None, inst, table [n,10], offs or None, pts or None)."""
        x = np.ascontiguousarray(img_u8, dtype=np.uint8)
        H, W, C = x.shape
        assert C == 3
        _, _, oc = self.out_shape(patch_in, patch_in)
        if max_rows is None:
            max_rows = max(16, H * W // 64)
        if pts_cap is None:
            pts_cap = max(4096, H * W // 16)

        def attempt():
            nonlocal max_rows, pts_cap
            pred = np.empty((H, W, oc), dtype=np.float32) if want_pred else None
            inst = np.empty((H, W), dtype=np.int32)
            table = np.zeros((max_rows, ROW_LEN), dtype=np.int64)
            nrows = np.zeros((1,), dtype=np.int32)
            offs = np.zeros((max_rows + 1,), dtype=np.int32) if contours else None
            pts = np.empty((pts_cap, 2), dtype=np.int32) if contours else None
            rc = self._retry_range(lambda: lib().hvn_infer_tile(
                self._h, _ptr(x), H, W, int(patch_in), int(batch), _ptr(pred), _ptr(inst), _ptr(table), int(max_rows),
                _ptr(nrows), _ptr(pts), int(pts_cap if contours else 0), _ptr(offs)))
            if rc == -4:
                if int(nrows[0]) > max_rows:
                    max_rows = int(nrows[0])
                else:
                    pts_cap = int(offs[-1])
            n = int(nrows[0])
            return rc, (pred, inst, table[:n], offs, (pts[: int(offs[-1])] if contours else None))
        return _retry_capacity("infer_tile", attempt)

    def infer_tiles(self, imgs, patch_in, batch=0, want_pred=True, contours=True, rows_cap=None, pts_cap=None,
                    features=False):
        """A group of RGB images [H_i,W_i,3] of any sizes through the device tile path in one stream of batches
        (hvn_infer_tiles).  Returns one (pred or None, inst, table [k,10], offs or None, pts or None) per image, each
        equal to infer_tile on that image alone; with features (needs contours) each tuple gains the image's
        inst_features rows [k,FEAT_LEN], measured on the group's device buffers (a TilesJob) before they are freed."""
        if features and not contours:
            raise ValueError("instance features need the contours")
        packed, shapes = pack_images(imgs)
        n = shapes.shape[0]
        if n < 1:
            raise ValueError("infer_tiles needs at least one image")
        if features:
            return TilesJob(self, list(imgs), patch_in, batch, want_pred, contours, True, rows_cap, pts_cap).result()
        px = int(packed.size // 3)
        _, _, oc = self.out_shape(patch_in, patch_in)
        r0, p0 = tiles_sizes(shapes)
        rows_cap = r0 if rows_cap is None else int(rows_cap)
        pts_cap = p0 if pts_cap is None else int(pts_cap)

        def attempt():  # a capacity failure grows the table once, then the point buffer once
            nonlocal rows_cap, pts_cap
            pred = np.empty((px * oc,), dtype=np.float32) if want_pred else None
            inst = np.empty((px,), dtype=np.int32)
            table = np.empty((rows_cap, ROW_LEN), dtype=np.int64)
            ro = np.zeros((n + 1,), dtype=np.int32)
            po = np.zeros((rows_cap + 1,), dtype=np.int32) if contours else None
            pts = np.empty((pts_cap, 2), dtype=np.int32) if contours else None
            rc = self._retry_range(lambda: lib().hvn_infer_tiles(
                self._h, n, _ptr(packed), _ptr(shapes), int(patch_in), int(batch), _ptr(pred), _ptr(inst), _ptr(table),
                int(rows_cap), _ptr(ro), _ptr(pts), int(pts_cap if contours else 0), _ptr(po)))
            rows = int(ro[-1])
            if rc == -4:
                if rows > rows_cap:
                    rows_cap = rows
                else:
                    pts_cap = int(po[rows])
                return rc, None
            if contours:
                po = po[: rows + 1]
                pts = pts[: int(po[-1])]
            return rc, (inst, table[:rows], ro, pred, pts, po)
        inst, table, ro, pred, pts, po = _retry_capacity("infer_tiles", attempt)
        return split_tiles(shapes, inst, table, ro, pred, pts, po)

    def infer_tiles_begin(self, imgs, patch_in, batch=0, want_pred=True, contours=True, features=False):
        """Enqueues a tile group with hvn_infer_tiles_dev and returns at once; TilesJob.result() waits for it."""
        return TilesJob(self, list(imgs), patch_in, batch, want_pred, contours, features)

    def infer_tiles_dev(self, n, d_imgs, shapes, patch_in, batch, d_pred, d_inst, d_table, rows_cap, d_row_offs, d_pts,
                        pts_cap, d_pt_offs):
        """hvn_infer_tiles_dev on device pointers (shapes: host int32 [n,2]); stream-ordered, no synchronisation."""
        sh = np.ascontiguousarray(shapes, dtype=np.int32)
        check(lib().hvn_infer_tiles_dev(self._h, int(n), _ptr(d_imgs), _ptr(sh), int(patch_in), int(batch), _ptr(d_pred),
                                        _ptr(d_inst), _ptr(d_table), int(rows_cap), _ptr(d_row_offs), _ptr(d_pts),
                                        int(pts_cap), _ptr(d_pt_offs)))

    def tile_predict_dev(self, d_img, H, W, patch_in, cell_lo, cell_hi, batch, d_pred):
        check(lib().hvn_tile_predict_dev(self._h, _ptr(d_img), int(H), int(W), int(patch_in), int(cell_lo), int(cell_hi),
                                         int(batch), _ptr(d_pred)))

    def forward_postproc(self, imgs_u8, want_pred=True, max_rows=None):
        x = np.ascontiguousarray(imgs_u8, dtype=np.uint8)
        B, H, W, _ = x.shape
        oh, ow, oc = self.out_shape(H, W)
        if max_rows is None:
            max_rows = max(16, oh * ow // 64)

        def attempt():
            nonlocal max_rows
            pred = np.empty((B, oh, ow, oc), dtype=np.float32) if want_pred else None
            inst = np.empty((B, oh, ow), dtype=np.int32)
            table = np.zeros((B, max_rows, ROW_LEN), dtype=np.int64)
            nrows = np.zeros((B,), dtype=np.int32)
            rc = self._retry_range(lambda: lib().hvn_forward_postproc(self._h, _ptr(x), B, H, W, _ptr(pred), _ptr(inst),
                                                                      _ptr(table), int(max_rows), _ptr(nrows)))
            if rc == -4:
                max_rows = int(nrows.max())
            return rc, (pred, inst, table, nrows)
        return _retry_capacity("forward_postproc", attempt)

    # ---- device-pointer entry points + helpers (bench / resident pipelines)
    def malloc(self, nbytes):
        p = ctypes.c_void_p()
        check(lib().hvn_malloc(self._h, int(nbytes), ctypes.byref(p)))
        return p.value

    def free(self, p):
        check(lib().hvn_free(self._h, ctypes.c_void_p(p)))

    def malloc_host(self, nbytes):
        p = ctypes.c_void_p()
        check(lib().hvn_malloc_host(self._h, int(nbytes), ctypes.byref(p)))
        return p.value

    def free_host(self, p):
        check(lib().hvn_free_host(self._h, ctypes.c_void_p(p)))

    def h2d(self, dst, src, nbytes):
        check(lib().hvn_memcpy_h2d(self._h, _ptr(dst), _ptr(src), int(nbytes)))

    def d2h(self, dst, src, nbytes):
        check(lib().hvn_memcpy_d2h(self._h, _ptr(dst), _ptr(src), int(nbytes)))

    def sync(self):
        check(lib().hvn_sync(self._h))

    def timer_start(self):
        check(lib().hvn_timer_start(self._h))

    def timer_stop(self):
        ms = ctypes.c_float()
        check(lib().hvn_timer_stop(self._h, ctypes.byref(ms)))
        return ms.value

    def stage_ms(self, name):
        ms = ctypes.c_float()
        check(lib().hvn_stage_ms(self._h, name.encode(), ctypes.byref(ms)))
        return ms.value

    def forward_dev(self, d_imgs, B, H, W, d_out):
        check(lib().hvn_forward_dev(self._h, _ptr(d_imgs), B, H, W, _ptr(d_out)))

    def postproc_dev(self, d_pred, n, H, W, C, nr_types, d_inst, d_table, max_rows, d_nrows):
        check(lib().hvn_postproc_dev(self._h, _ptr(d_pred), n, H, W, C, int(nr_types or 0), _ptr(d_inst),
                                     _ptr(d_table), int(max_rows), _ptr(d_nrows)))

    def pack_tables_dev(self, d_table, d_nrows, n, max_rows, d_packed, cap_rows, d_offs):
        """padded tables [n,max_rows,10] -> packed rows [<=cap_rows,10] + offs [n+1] (all device pointers)."""
        check(lib().hvn_pack_tables_dev(self._h, _ptr(d_table), _ptr(d_nrows), int(n), int(max_rows), _ptr(d_packed),
                                        int(cap_rows), _ptr(d_offs)))

    def stream_handle(self):
        """The context's cudaStream_t as an integer (e.g. for torch.cuda.ExternalStream)."""
        p = ctypes.c_void_p()
        check(lib().hvn_get_stream(self._h, ctypes.byref(p)))
        return int(p.value or 0)

    def forward_postproc_dev(self, d_imgs, B, H, W, d_pred, d_inst, d_table, max_rows, d_nrows):
        check(lib().hvn_forward_postproc_dev(self._h, _ptr(d_imgs), B, H, W, _ptr(d_pred), _ptr(d_inst),
                                             _ptr(d_table), int(max_rows), _ptr(d_nrows)))
