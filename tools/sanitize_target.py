"""Small end-to-end run for compute-sanitizer (memcheck / racecheck / synccheck / initcheck): 1 patch through CNN +
post-processing (every k_conv_tc variant the plan uses -- plain, XF transform, residual, two-source, upsample -- and the
tensor-core stem), device contours, the whole-image tile path on a small image, the packed
table gather kernel, and a 300x200 synthetic map through the generic (large-map) flood.
HVN_SAN_MODE=original runs the 270x270 / 5x5 variant of the CNN part only; HVN_SAN_CNN_ONLY=1 stops
the fast-mode run after the CNN + post-processing pass; HVN_SAN_REFEREE=1 adds the CUDA-core referee."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from hover_net_b200 import synth
from hover_net_b200.models.hovernet.net_desc import create_model

if os.environ.get("HVN_SAN_MODE") == "original":
    net = create_model(mode="original", nr_types=5)
    net.load_state_dict(synth.make_state_dict("original", 5, 0))
    x = synth.make_patches(1, 270, seed=1)
    pred, inst, tab, n = net.ctx.forward_postproc(x)
    print("tc path (original) ok", int(n[0]), bool(np.isfinite(pred).all()))
    net.ctx.close()
    sys.exit(0)
net = create_model(mode="fast", nr_types=6)
net.load_state_dict(synth.make_state_dict("fast", 6, 0))
x = synth.make_patches(1, 256, seed=1)
pred, inst, tab, n = net.ctx.forward_postproc(x)
print("tc path ok", int(n[0]))
if os.environ.get("HVN_SAN_CNN_ONLY"):   # the kernels of csrc/conv_tc.cu only (k_conv_tc variants, stem)
    net.ctx.close()
    sys.exit(0)
pm = synth.synth_pred_map(164, 164, 6, 0)
gi, gt, gn, offs, pts = net.ctx.postproc_contours(pm, 6)
print("contours ok", int(gn[0]), len(pts))
img = np.concatenate([x[0], x[0][:, ::-1]], 1)[:200, :300]
tp, ti, tt, toffs, tpts = net.ctx.infer_tile(img, 256, 4)
print("tile path ok", len(tt), len(tpts))
if os.environ.get("HVN_SAN_REFEREE"):
    net.ctx.set_option("conv_path", 1)
    pred2 = net.ctx.forward(x)
    print("referee path ok", float(np.abs(pred2[..., 1:] - pred[..., 1:]).max()))
pm = synth.synth_pred_map(300, 200, 6, 0)
net.ctx.set_option("flood_impl", 2)
gi, gt, gn = net.ctx.postproc(pm, 6)
print("generic flood ok", int(gn[0]))
net.ctx.close()
