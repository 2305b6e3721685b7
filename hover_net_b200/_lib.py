"""ctypes binding of libhvn.so (include/hvn.h).  There is no CPU fallback: if the CUDA library is
missing or no sm_90 device is present, every entry point raises."""
import ctypes
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libhvn.so")
ROW_LEN = 10
_lib = None


class HvnError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("libhvn error %d: %s" % (code, msg))
        self.code = code


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise HvnError(-2, "libhvn.so is not built (run `python -c 'import __graft_entry__ as g; g.build()'`); "
                               "this package has no CPU fallback")
        L = ctypes.CDLL(LIB_PATH)
        L.hvn_last_error.restype = ctypes.c_char_p
        L.hvn_debug_log.restype = ctypes.c_char_p
        L.hvn_debug_log.argtypes = [ctypes.c_void_p]
        L.hvn_get_counter.restype = ctypes.c_int64
        L.hvn_get_counter.argtypes = [ctypes.c_void_p, ctypes.c_char_p]
        L.hvn_set_option.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_int64]
        for name in ("hvn_malloc", "hvn_malloc_host"):
            getattr(L, name).argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.POINTER(ctypes.c_void_p)]
        for name in ("hvn_memcpy_h2d", "hvn_memcpy_d2h"):
            getattr(L, name).argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t]
        for name in ("hvn_free", "hvn_free_host"):
            getattr(L, name).argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        _lib = L
    return _lib


def check(rc):
    if rc != 0:
        raise HvnError(rc, lib().hvn_last_error().decode("utf-8", "replace"))


def _ptr(a):
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        return a.ctypes.data_as(ctypes.c_void_p)
    return ctypes.c_void_p(int(a))  # raw address (device pointer or pinned host)


def _as_ids(a):
    """Instance map as C-contiguous int32; ids that int32 cannot hold are an error, never wrapped."""
    a = np.asarray(a)
    if a.dtype == np.int32:
        return np.ascontiguousarray(a)
    b = np.ascontiguousarray(a, dtype=np.int32)
    if not np.array_equal(b, a):
        raise ValueError("instance ids must be integers that fit in int32")
    return b


class Context:
    """One libhvn context (one device, one stream)."""

    def __init__(self, device=0, mode=None, nr_types=None):
        self._h = ctypes.c_void_p()
        L = lib()
        if mode is None:
            check(L.hvn_create_postproc(int(device), ctypes.byref(self._h)))
        else:
            check(L.hvn_create(int(device), mode.encode(), int(nr_types or 0), ctypes.byref(self._h)))
        self.device = int(device)
        self.mode = mode
        self.nr_types = nr_types
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
        while True:
            inst = np.empty((n, H, W), dtype=np.int32)
            table = np.zeros((n, max_rows, ROW_LEN), dtype=np.int64)
            nrows = np.zeros((n,), dtype=np.int32)
            rc = lib().hvn_postproc(self._h, _ptr(p), n, H, W, C, int(nr_types or 0), _ptr(inst), _ptr(table),
                                    int(max_rows), _ptr(nrows))
            if rc == -4:  # HVN_ERR_CAPACITY: retry with the exact size
                max_rows = int(nrows.max())
                continue
            check(rc)
            return inst, table, nrows

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
        for _attempt in range(4):  # at most: grow the table once, then the point buffer once
            inst = np.empty((n, H, W), dtype=np.int32)
            table = np.zeros((n, max_rows, ROW_LEN), dtype=np.int64)
            nrows = np.zeros((n,), dtype=np.int32)
            offs = np.zeros((n * max_rows + 1,), dtype=np.int32)
            pts = np.empty((pts_cap, 2), dtype=np.int32)
            L = lib()
            L.hvn_postproc_contours.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                                ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int,
                                                ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p]
            rc = L.hvn_postproc_contours(self._h, _ptr(p), n, H, W, C, int(nr_types or 0), _ptr(inst), _ptr(table),
                                         int(max_rows), _ptr(nrows), _ptr(pts), int(pts_cap), _ptr(offs))
            if rc == -4:  # HVN_ERR_CAPACITY: the table or the point buffer was too small -- retry with exact sizes
                if int(nrows.max()) > max_rows:
                    max_rows = int(nrows.max())
                else:
                    pts_cap = int(offs[-1])
                continue
            check(rc)
            return inst, table, nrows, offs, pts[: int(offs[-1])]
        raise HvnError(-4, "postproc_contours: capacity retries exhausted")

    def contours_dev(self, d_inst, d_table, d_nrows, n, H, W, max_rows, d_pts, pts_cap, d_offs):
        L = lib()
        L.hvn_contours_dev.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int,
                                       ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p]
        check(L.hvn_contours_dev(self._h, _ptr(d_inst), _ptr(d_table), _ptr(d_nrows), n, H, W, int(max_rows), _ptr(d_pts),
                                 int(pts_cap), _ptr(d_offs)))

    _PAIRS_ARGS = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                   ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p]

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
        L = lib()
        L.hvn_inst_pairs.argtypes = self._PAIRS_ARGS
        for _attempt in range(2):
            rows = np.empty((cap, 3), dtype=np.int64)
            offs = np.zeros((n + 1,), dtype=np.int64)
            rc = L.hvn_inst_pairs(self._h, _ptr(t), _ptr(p), n, H, W, _ptr(rows), int(cap), _ptr(offs))
            if rc == -4:  # HVN_ERR_CAPACITY: retry with the exact size
                cap = int(offs[-1])
                continue
            check(rc)
            rows = rows[: int(offs[-1])]
            m = np.repeat(np.arange(n), np.diff(offs))
            return rows[np.lexsort((rows[:, 1], rows[:, 0], m))], offs
        raise HvnError(-4, "inst_pairs: capacity retries exhausted")

    def inst_pairs_dev(self, d_true, d_pred, n, H, W, d_pairs, cap, d_offs):
        """Device-pointer variant (d_pred may be None).  Returns False on HVN_ERR_CAPACITY (offs is valid on the
        device then: retry with cap >= offs[n]), True on success; raises on any other error."""
        L = lib()
        L.hvn_inst_pairs_dev.argtypes = self._PAIRS_ARGS
        rc = L.hvn_inst_pairs_dev(self._h, _ptr(d_true), _ptr(d_pred), int(n), int(H), int(W), _ptr(d_pairs),
                                  int(cap), _ptr(d_offs))
        if rc == -4:
            return False
        check(rc)
        return True

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
        L = lib()
        L.hvn_infer_tile.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                     ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p,
                                     ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p]
        for _attempt in range(4):
            pred = np.empty((H, W, oc), dtype=np.float32) if want_pred else None
            inst = np.empty((H, W), dtype=np.int32)
            table = np.zeros((max_rows, ROW_LEN), dtype=np.int64)
            nrows = np.zeros((1,), dtype=np.int32)
            offs = np.zeros((max_rows + 1,), dtype=np.int32) if contours else None
            pts = np.empty((pts_cap, 2), dtype=np.int32) if contours else None
            rc = self._retry_range(lambda: L.hvn_infer_tile(
                self._h, _ptr(x), H, W, int(patch_in), int(batch), _ptr(pred), _ptr(inst), _ptr(table), int(max_rows),
                _ptr(nrows), _ptr(pts), int(pts_cap if contours else 0), _ptr(offs)))
            if rc == -4:
                if int(nrows[0]) > max_rows:
                    max_rows = int(nrows[0])
                else:
                    pts_cap = int(offs[-1])
                continue
            check(rc)
            n = int(nrows[0])
            return pred, inst, table[:n], offs, (pts[: int(offs[-1])] if contours else None)
        raise HvnError(-4, "infer_tile: capacity retries exhausted")

    def tile_predict_dev(self, d_img, H, W, patch_in, cell_lo, cell_hi, batch, d_pred):
        L = lib()
        L.hvn_tile_predict_dev.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                           ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
        check(L.hvn_tile_predict_dev(self._h, _ptr(d_img), int(H), int(W), int(patch_in), int(cell_lo), int(cell_hi),
                                     int(batch), _ptr(d_pred)))

    def forward_postproc(self, imgs_u8, want_pred=True, max_rows=None):
        x = np.ascontiguousarray(imgs_u8, dtype=np.uint8)
        B, H, W, _ = x.shape
        oh, ow, oc = self.out_shape(H, W)
        if max_rows is None:
            max_rows = max(16, oh * ow // 64)
        while True:
            pred = np.empty((B, oh, ow, oc), dtype=np.float32) if want_pred else None
            inst = np.empty((B, oh, ow), dtype=np.int32)
            table = np.zeros((B, max_rows, ROW_LEN), dtype=np.int64)
            nrows = np.zeros((B,), dtype=np.int32)
            rc = self._retry_range(lambda: lib().hvn_forward_postproc(self._h, _ptr(x), B, H, W, _ptr(pred), _ptr(inst),
                                                                      _ptr(table), int(max_rows), _ptr(nrows)))
            if rc == -4:
                max_rows = int(nrows.max())
                continue
            check(rc)
            return pred, inst, table, nrows

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
        L = lib()
        L.hvn_pack_tables_dev.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                          ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p]
        check(L.hvn_pack_tables_dev(self._h, _ptr(d_table), _ptr(d_nrows), int(n), int(max_rows), _ptr(d_packed),
                                    int(cap_rows), _ptr(d_offs)))

    def stream_handle(self):
        """The context's cudaStream_t as an integer (e.g. for torch.cuda.ExternalStream)."""
        p = ctypes.c_void_p()
        L = lib()
        L.hvn_get_stream.argtypes = [ctypes.c_void_p, ctypes.POINTER(ctypes.c_void_p)]
        check(L.hvn_get_stream(self._h, ctypes.byref(p)))
        return int(p.value or 0)

    def forward_postproc_dev(self, d_imgs, B, H, W, d_pred, d_inst, d_table, max_rows, d_nrows):
        check(lib().hvn_forward_postproc_dev(self._h, _ptr(d_imgs), B, H, W, _ptr(d_pred), _ptr(d_inst),
                                             _ptr(d_table), int(max_rows), _ptr(d_nrows)))
