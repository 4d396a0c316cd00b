"""CPU test: every C-ABI entry point's argument checks, one function at a time.

For each function of include/msda_b200.h there is one valid call.  It must get past the checks (neither MSDA_E_BADARG
nor MSDA_E_TOOLARGE); an early return (nothing to do: I == 0, planes == 0, B == 0, ...) must return exactly 0.  Each
required pointer set to NULL must give MSDA_E_BADARG, and each documented limit its documented code.  The pure host
functions (workspace sizes, routing predicates) must return the recorded values.

The calls use fake, 4 KiB-aligned device addresses.  Without a GPU a call that passes the checks fails in the CUDA
runtime with a positive code; on a machine with a GPU it would launch kernels on the fake addresses, so the file is
skipped there."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.skipif(torch.cuda.is_available(), reason="calls with fake device addresses")

BADARG, TOOLARGE = -1, -2
BASE = 0x7F0000000000                           # one 1 MiB slot per pointer operand
BIG_WS = 1 << 40                                # workspace_bytes large enough for every valid call below


class Spec:
    """ptrs: pointer operands in argument order; optional: those that may be NULL; sizes: the valid call's sizes;
    args(p, s): the argument list; limits: (size overrides, expected code); early: size overrides that return 0."""

    def __init__(self, ptrs, sizes, args, optional=(), limits=(), early=()):
        self.ptrs, self.sizes, self.args = ptrs, sizes, args
        self.optional, self.limits, self.early = set(optional), list(limits), list(early)

    def call(self, lib, fn, null=None, **over):
        out = ctypes.c_int64(-7)                # `bytes` of the workspace queries is written on the host
        p = {n: (None if n == null else ctypes.addressof(out) if n == "bytes" else BASE + (i << 20))
             for i, n in enumerate(self.ptrs)}
        return getattr(lib, fn)(*self.args(p, dict(self.sizes, **over)))


def _nonpos(*names):
    return [({n: v}, BADARG) for n in names for v in (0, -1)]


# ---- the op -----------------------------------------------------------------------------------------------------------
OP = dict(N=2, S=64, M=2, D=32, L=2, Lq=10, P=4)
OP_LIMITS = _nonpos(*OP) + [
    (dict(S=1 << 30), TOOLARGE),                                        # rows are int32 within a batch element
    (dict(N=1 << 10, Lq=1 << 20, M=1 << 10), TOOLARGE),                 # N * Lq * M >= 2^40
    (dict(N=1 << 10, Lq=(1 << 20) - 1, M=1 << 10, D=3), 0),             # just below: passes (generic route)
]
OP_FWD = ("value", "shapes", "lsi", "loc", "attn", "out")
OP_BWD = ("grad_out", "value", "shapes", "lsi", "loc", "attn", "gv", "gl", "ga")
OP_BWD16 = ("grad_out", "value", "shapes", "lsi", "loc", "attn", "gv32", "gv", "gl", "ga")
_dims = lambda s: (s["N"], s["S"], s["M"], s["D"], s["L"], s["Lq"], s["P"])
DET_LIMITS = OP_LIMITS[:-1] + [
    (dict(M=8, S=1 << 29), TOOLARGE),                                   # M * S + 1 > 2^32: 32-bit keys and sentinel
    (dict(M=8, S=(1 << 29) - 1), 0),
    (dict(M=1 << 12, L=1 << 12, P=1 << 8), TOOLARGE),                   # one query's M*L*P*4 entries > 2^32 - 1
    (dict(ws_bytes=0), BADARG), (dict(ws_bytes=-1), BADARG),
]


def _det(ptrs):
    def args(p, s):
        return tuple(p[n] for n in ptrs[:6]) + _dims(s) + tuple(p[n] for n in ptrs[6:]) + (s.get("ws_bytes", BIG_WS), None)
    return args


SPECS = {
    "msda_forward_f32": Spec(OP_FWD, OP, lambda p, s: (p["value"], p["shapes"], p["lsi"], p["loc"], p["attn"]) + _dims(s)
                             + (p["out"], None), limits=OP_LIMITS),
    "msda_forward_f64": Spec(OP_FWD, OP, lambda p, s: (p["value"], p["shapes"], p["lsi"], p["loc"], p["attn"]) + _dims(s)
                             + (p["out"], None), limits=OP_LIMITS),
    "msda_forward_bf16": Spec(OP_FWD, OP, lambda p, s: (p["value"], p["shapes"], p["lsi"], p["loc"], p["attn"]) + _dims(s)
                              + (p["out"], None), limits=OP_LIMITS),
    "msda_backward_f32": Spec(OP_BWD, OP, lambda p, s: tuple(p[n] for n in OP_BWD[:6]) + _dims(s)
                              + (p["gv"], p["gl"], p["ga"], None), limits=OP_LIMITS),
    "msda_backward_f64": Spec(OP_BWD, OP, lambda p, s: tuple(p[n] for n in OP_BWD[:6]) + _dims(s)
                              + (p["gv"], p["gl"], p["ga"], None), limits=OP_LIMITS),
    "msda_backward_bf16": Spec(OP_BWD16, OP, lambda p, s: tuple(p[n] for n in OP_BWD16[:6]) + _dims(s)
                               + (p["gv32"], p["gv"], p["gl"], p["ga"], None), optional=("gv",), limits=OP_LIMITS),
    "msda_backward_det_f32": Spec(OP_BWD + ("ws",), OP, _det(OP_BWD + ("ws",)), limits=DET_LIMITS),
    "msda_backward_det_f64": Spec(OP_BWD + ("ws",), OP, _det(OP_BWD + ("ws",)), limits=DET_LIMITS),
    "msda_backward_det_bf16": Spec(OP_BWD16 + ("ws",), OP, _det(OP_BWD16 + ("ws",)), optional=("gv",),
                                   limits=DET_LIMITS),
    "msda_backward_det_workspace": Spec(
        ("bytes",), dict(OP, dt=4, chunk=4),
        lambda p, s: (s["dt"],) + _dims(s) + (s["chunk"], p["bytes"]),
        limits=[(dict(dt=1), BADARG), (dict(dt=3), BADARG), (dict(chunk=0), BADARG), (dict(chunk=-1), BADARG)]
        + [lim for lim in DET_LIMITS if "ws_bytes" not in lim[0]]),
}

# ---- callers of the op ------------------------------------------------------------------------------------------------
PRO = dict(R=6, M=2, L=2, P=3, refdim=2)
PRO_LIMITS = _nonpos("R", "M", "L", "P") + [(dict(L=4, P=9), BADARG), (dict(L=4, P=8), 0), (dict(refdim=3), BADARG),
                                             (dict(refdim=4), 0)]
SPECS.update({
    "msda_prologue_forward_f32": Spec(
        ("proj", "ref", "shapes", "loc", "attn"), PRO,
        lambda p, s: (p["proj"], p["ref"], p["shapes"], s["R"], s["M"], s["L"], s["P"], s["refdim"], p["loc"], p["attn"],
                      None),
        limits=PRO_LIMITS + [(dict(R=1 << 30, M=1 << 5), BADARG), (dict(R=1 << 30, M=(1 << 5) - 1), 0)]),
    "msda_prologue_backward_f32": Spec(
        ("grad_loc", "grad_attn", "attn", "ref", "shapes", "grad_proj"), PRO,
        lambda p, s: (p["grad_loc"], p["grad_attn"], p["attn"], p["ref"], p["shapes"], s["R"], s["M"], s["L"], s["P"],
                      s["refdim"], p["grad_proj"], None),
        limits=PRO_LIMITS),
    "msda_colsum_f32": Spec(("x", "out"), dict(rows=10, cols=256),
                            lambda p, s: (p["x"], s["rows"], s["cols"], p["out"], None),
                            limits=_nonpos("rows", "cols") + [(dict(cols=258), BADARG)]),
    "msda_relu_backward_colsum_f32": Spec(
        ("g", "y", "g2", "colsum"), dict(rows=10, cols=256),
        lambda p, s: (p["g"], p["y"], s["rows"], s["cols"], p["g2"], p["colsum"], None),
        limits=_nonpos("rows", "cols") + [(dict(cols=6), BADARG)]),
    "msda_add_layernorm_forward_f32": Spec(
        ("a", "b", "gamma", "beta", "z", "y", "mean", "rstd"), dict(rows=10, cols=256),
        lambda p, s: (p["a"], p["b"], p["gamma"], p["beta"], s["rows"], s["cols"], 1e-5, p["z"], p["y"], p["mean"],
                      p["rstd"], None),
        optional=("b",), limits=_nonpos("rows") + [(dict(cols=c), BADARG) for c in (0, 64, 320, 640)]
        + [(dict(cols=c), 0) for c in (128, 384, 512)]),
    "msda_layernorm_backward_f32": Spec(
        ("dy", "z", "gamma", "mean", "rstd", "dz", "dgamma", "dbeta"), dict(rows=10, cols=128),
        lambda p, s: (p["dy"], p["z"], p["gamma"], p["mean"], p["rstd"], s["rows"], s["cols"], p["dz"], p["dgamma"],
                      p["dbeta"], None),
        limits=_nonpos("rows") + [(dict(cols=c), BADARG) for c in (0, 130, 1024)]),
    "msda_linear_tf32": Spec(
        ("A", "W", "bias", "C"), dict(M=100, N=384, K=256),
        lambda p, s: (p["A"], p["W"], p["bias"], s["M"], s["N"], s["K"], p["C"], None),
        optional=("bias",),
        limits=_nonpos("M", "N", "K") + [(dict(K=48), BADARG), (dict(N=48), BADARG), (dict(N=544), BADARG),
                                         (dict(N=288), BADARG), (dict(N=32), 0), (dict(N=512), 0)]),
    "msda_linear_tf32_ex": Spec(
        ("A", "W", "bias", "row_mask", "C"), dict(M=100, N=256, K=256),
        lambda p, s: (p["A"], p["W"], p["bias"], p["row_mask"], s["M"], s["N"], s["K"], 1, p["C"], None),
        optional=("bias", "row_mask"),
        limits=_nonpos("M", "N", "K") + [(dict(N=32), BADARG), (dict(N=96), BADARG), (dict(N=320), BADARG),
                                         (dict(K=48), BADARG), (dict(N=64), 0)]),
})

# ---- geometry feeding the op ------------------------------------------------------------------------------------------
GEO = dict(N=2, S=64, L=2)
SPECS.update({
    "msda_valid_counts": Spec(("mask", "shapes", "lsi", "counts"), GEO,
                              lambda p, s: (p["mask"], p["shapes"], p["lsi"], s["N"], s["S"], s["L"], p["counts"], None),
                              limits=_nonpos("N", "S", "L")),
    "msda_encoder_ref_points_f32": Spec(
        ("ratios", "shapes", "lsi", "ref"), GEO,
        lambda p, s: (p["ratios"], p["shapes"], p["lsi"], s["N"], s["S"], s["L"], p["ref"], None),
        limits=_nonpos("N", "S", "L")),
    "msda_encoder_proposals_f32": Spec(
        ("mask", "counts", "shapes", "lsi", "proposals", "keep"), GEO,
        lambda p, s: (p["mask"], p["counts"], p["shapes"], p["lsi"], s["N"], s["S"], s["L"], 0.05, p["proposals"],
                      p["keep"], None),
        limits=_nonpos("N", "S", "L") + [(dict(L=31), BADARG), (dict(L=30), 0)]),
    "msda_sine_pos_embed_forward_f32": Spec(
        ("pos", "out"), dict(R=10, n=4, F=128),
        lambda p, s: (p["pos"], s["R"], s["n"], s["F"], 10000.0, 1, p["out"], None), limits=_nonpos("R", "n", "F")),
    "msda_sine_pos_embed_backward_f32": Spec(
        ("pos", "grad_out", "grad_pos"), dict(R=10, n=4, F=128),
        lambda p, s: (p["pos"], p["grad_out"], s["R"], s["n"], s["F"], 10000.0, 1, p["grad_pos"], None),
        limits=_nonpos("R", "n", "F")),
})

# ---- CondInst ---------------------------------------------------------------------------------------------------------
CI = dict(N=2, H=40, W=64, I=5, max_inst=3, stride=8)
CI_LIMITS = _nonpos("N", "H", "W", "stride") + [(dict(I=-1), BADARG), (dict(max_inst=-1), BADARG),
                                                 (dict(H=1 << 15, W=1 << 15), BADARG), (dict(H=1 << 15, W=(1 << 15) - 1), 0)]
AB = dict(planes=6, h=13, w=21, factor=2)
AB_LIMITS = _nonpos("h", "w", "factor") + [(dict(planes=-1), BADARG), (dict(planes=1 << 31), BADARG),
                                           (dict(h=1 << 15, w=1 << 14, factor=2), BADARG),     # output >= 2^31 pixels
                                           (dict(h=1 << 15, w=(1 << 14) - 1, factor=2), 0)]
SPECS.update({
    "msda_condinst_forward_f32": Spec(
        ("feats", "params", "refs", "inst_start", "logits"), CI,
        lambda p, s: (p["feats"], p["params"], p["refs"], p["inst_start"], s["N"], s["H"], s["W"], s["I"], s["max_inst"],
                      s["stride"], 1, p["logits"], None),
        limits=CI_LIMITS, early=[dict(I=0), dict(max_inst=0)]),
    "msda_condinst_backward_f32": Spec(
        ("grad_logits", "feats", "params", "refs", "inst_start", "grad_feats", "grad_params", "grad_refs"), CI,
        lambda p, s: (p["grad_logits"], p["feats"], p["params"], p["refs"], p["inst_start"], s["N"], s["H"], s["W"],
                      s["I"], s["max_inst"], s["stride"], 1, p["grad_feats"], p["grad_params"], p["grad_refs"], None),
        limits=CI_LIMITS + [(dict(I=0), 0), (dict(max_inst=0), 0)]),       # zero-fills grad_feats first
    "msda_aligned_bilinear_forward_f32": Spec(
        ("in", "out"), AB, lambda p, s: (p["in"], s["planes"], s["h"], s["w"], s["factor"], p["out"], None),
        limits=AB_LIMITS, early=[dict(planes=0)]),
    "msda_aligned_bilinear_backward_f32": Spec(
        ("grad_out", "grad_in"), AB, lambda p, s: (p["grad_out"], s["planes"], s["h"], s["w"], s["factor"], p["grad_in"],
                                                   None),
        limits=AB_LIMITS, early=[dict(planes=0)]),
})

# ---- mask pasting, COCO RLE, detection post-processing ----------------------------------------------------------------
MP = dict(I=3, Hs=20, Ws=30, stride=4, crop_h=70, crop_w=110, out_h=300, out_w=500)
MP_LIMITS = _nonpos("Hs", "Ws", "stride", "crop_h", "crop_w", "out_h", "out_w") + [
    (dict(I=-1), BADARG),
    (dict(stride=1 << 26, Hs=32), BADARG), (dict(stride=1 << 26, Ws=32), BADARG),      # stride * Hs >= 2^31
    (dict(crop_h=81), BADARG), (dict(crop_w=121), BADARG), (dict(crop_h=80, crop_w=120), 0),
    (dict(out_h=65535 * 16 + 1, out_w=1), TOOLARGE), (dict(out_h=65535 * 16, out_w=1), 0),
]
RLE_LIMITS = [(dict(out_h=0), BADARG), (dict(out_w=0), BADARG), (dict(I=-1), BADARG),
              (dict(I=1 << 31), TOOLARGE), (dict(out_h=1 << 16, out_w=(1 << 16) + 1), TOOLARGE),
              (dict(out_h=1, out_w=1 << 30), TOOLARGE)]
DP = dict(B=2, Q=300, T=256, C=80, max_num_inst=100)
DP_LIMITS = [(dict(B=-1), BADARG), (dict(B=65536), BADARG), (dict(Q=0), BADARG), (dict(Q=1025), BADARG),
             (dict(T=0), BADARG), (dict(T=257), BADARG), (dict(C=0), BADARG), (dict(C=4097), BADARG),
             (dict(max_num_inst=0), BADARG), (dict(Q=2, C=3, max_num_inst=7), BADARG), (dict(Q=2, C=3, max_num_inst=6), 0)]
DP_PTRS = ("box_cls", "box_pred", "iou_pred", "class_start", "tokens", "image_sizes", "scores", "labels", "query_index",
           "boxes", "count", "ws")
SPECS.update({
    "msda_mask_paste_f32": Spec(
        ("logits", "out"), dict(MP, binary=1),
        lambda p, s: (p["logits"], s["I"], s["Hs"], s["Ws"], s["stride"], s["crop_h"], s["crop_w"], s["out_h"],
                      s["out_w"], 0.5, s["binary"], p["out"], None),
        limits=MP_LIMITS + [(dict(out_w=1 << 30), TOOLARGE), (dict(binary=0), 0)], early=[dict(I=0)]),
    "msda_mask_rle_count_f32": Spec(
        ("logits", "ws"), dict(MP, ws_bytes=BIG_WS),
        lambda p, s: (p["logits"], s["I"], s["Hs"], s["Ws"], s["stride"], s["crop_h"], s["crop_w"], s["out_h"],
                      s["out_w"], 0.5, p["ws"], s["ws_bytes"], None),
        limits=MP_LIMITS + [(dict(I=1 << 31), TOOLARGE), (dict(out_h=1 << 16, out_w=(1 << 16) + 1), TOOLARGE),
                            (dict(out_w=1 << 30), TOOLARGE)],
        early=[dict(I=0)]),
    "msda_mask_rle_count_u8": Spec(
        ("masks", "ws"), dict(I=3, out_h=300, out_w=500, ws_bytes=BIG_WS),
        lambda p, s: (p["masks"], s["I"], s["out_h"], s["out_w"], p["ws"], s["ws_bytes"], None),
        limits=RLE_LIMITS, early=[dict(I=0)]),
    "msda_mask_rle_encode": Spec(
        ("ws", "positions", "byte_offsets", "chars"), dict(I=3, out_h=300, out_w=500, boundaries=1000, ws_bytes=BIG_WS),
        lambda p, s: (s["I"], s["out_h"], s["out_w"], s["boundaries"], p["ws"], s["ws_bytes"], p["positions"],
                      p["byte_offsets"], p["chars"], None),
        limits=RLE_LIMITS + [(dict(boundaries=-1), BADARG), (dict(boundaries=3 * 300 * 500 + 1), BADARG),
                             (dict(boundaries=3 * 300 * 500), 0)],
        early=[dict(I=0, boundaries=0)]),
    "msda_mask_rle_workspace": Spec(
        ("bytes",), dict(I=3, out_h=300, out_w=500),
        lambda p, s: (s["I"], s["out_h"], s["out_w"], p["bytes"]), limits=RLE_LIMITS),
    "msda_detpost_workspace": Spec(
        ("bytes",), DP, lambda p, s: (s["B"], s["Q"], s["T"], s["C"], s["max_num_inst"], p["bytes"]),
        limits=DP_LIMITS + [(dict(B=0), 0)]),
    "msda_detpost_f32": Spec(
        DP_PTRS, dict(DP, nms=1, ws_bytes=BIG_WS),
        lambda p, s: tuple(p[n] for n in DP_PTRS[:6]) + (s["B"], s["Q"], s["T"], s["C"], s["nms"], 0.7,
                                                         s["max_num_inst"]) + tuple(p[n] for n in DP_PTRS[6:])
        + (s["ws_bytes"], None),
        optional=("iou_pred",), limits=DP_LIMITS + [(dict(nms=0), 0), (dict(ws_bytes=0), BADARG)],
        early=[dict(B=0)]),
})

# ---- early-fusion attention -------------------------------------------------------------------------------------------
VLF = dict(B=2, H=8, S=300, T=32, hd=128, p=0.1)
VLF_SIZES = lambda s: (s["B"], s["H"], s["S"], s["T"], s["hd"])
VLF_LIMITS = _nonpos("B", "H", "S", "T") + [
    (dict(T=257), BADARG), (dict(T=256), 0), (dict(hd=64), BADARG), (dict(hd=192), BADARG), (dict(hd=256), 0),
    (dict(B=1 << 10, S=1 << 20, H=8, hd=128), TOOLARGE),                    # B * S * H * D >= 2^40
    (dict(B=1 << 10, H=64), TOOLARGE), (dict(B=1, S=1 << 30), TOOLARGE),
]
VLF_FWD = ("q", "k", "v_v", "v_l", "text_bias", "seed", "out_v", "out_l", "stats", "ws")
VLF_BWD = ("grad_out_v", "grad_out_l", "q", "k", "v_v", "v_l", "text_bias", "out_v", "out_l", "stats", "seed",
           "grad_q", "grad_k", "grad_v_v", "grad_v_l", "ws")
_vlf_dropout = [(dict(p=-0.1), BADARG), (dict(p=1.0), BADARG), (dict(p=float("nan")), BADARG), (dict(p=0.0), 0),
                (dict(ws_bytes=1024), BADARG)]
_vlf_fwd = Spec(VLF_FWD, dict(VLF, ws_bytes=BIG_WS),
                lambda p, s: tuple(p[n] for n in VLF_FWD[:5]) + VLF_SIZES(s) + (1, 1, s["p"], p["seed"])
                + tuple(p[n] for n in VLF_FWD[6:]) + (s["ws_bytes"], None),
                optional=("text_bias",), limits=VLF_LIMITS + _vlf_dropout)
_vlf_bwd = Spec(VLF_BWD, dict(VLF, ws_bytes=BIG_WS),
                lambda p, s: tuple(p[n] for n in VLF_BWD[:10]) + VLF_SIZES(s) + (1, 1, s["p"], p["seed"])
                + tuple(p[n] for n in VLF_BWD[11:]) + (s["ws_bytes"], None),
                optional=("text_bias",), limits=VLF_LIMITS + _vlf_dropout)
SPECS.update({f"msda_vlfuse_{d}_{m}": (_vlf_fwd if d == "forward" else _vlf_bwd)
              for d in ("forward", "backward") for m in ("f32", "tf32", "bf16")})
SPECS.update({
    "msda_vlfuse_workspace": Spec(("bytes",), VLF, lambda p, s: VLF_SIZES(s) + (p["bytes"],), limits=VLF_LIMITS),
    "msda_vlfuse_dropout_mask_f32": Spec(
        ("seed", "mask_v", "mask_l"), VLF,
        lambda p, s: (p["seed"], s["B"], s["H"], s["S"], s["T"], s["p"], p["mask_v"], p["mask_l"], None),
        limits=_nonpos("B", "H", "S", "T") + _vlf_dropout[:4]),
})

# ---- pure host functions: values recorded from the library ------------------------------------------------------------
WORKSPACE = [  # (function, sizes) -> bytes.  The det and RLE workspaces ask CUB, which needs a device: only I = 0 here
    ("msda_detpost_workspace", (2, 300, 256, 80, 100), 197120),
    ("msda_detpost_workspace", (0, 300, 256, 80, 100), 0),
    ("msda_detpost_workspace", (1, 900, 256, 1203, 3000), 4371456),
    ("msda_detpost_workspace", (4, 1024, 1, 4096, 2048), 67141632),
    ("msda_detpost_workspace", (3, 1024, 1, 4096, 2049), 50454528),      # past 2048: a sort buffer in the workspace
    ("msda_mask_rle_workspace", (0, 300, 500), 0),
    ("msda_vlfuse_workspace", (2, 8, 300, 32, 128), 1069824),
    ("msda_vlfuse_workspace", (1, 8, 22323, 256, 256), 63637248),
    ("msda_vlfuse_workspace", (2, 1, 17, 1, 128), 2560),
    ("msda_vlfuse_workspace", (4, 8, 13101, 256, 256), 68818688),
]
FAST_PATH = [  # (dtype_bytes, D, L, P) -> msda_uses_fast_path
    ((4, 16, 4, 4), 1), ((4, 32, 4, 4), 1), ((4, 64, 4, 8), 1), ((4, 32, 8, 4), 1), ((4, 32, 9, 1), 0),
    ((4, 32, 4, 9), 0), ((4, 8, 4, 4), 0), ((4, 128, 4, 4), 0), ((4, 30, 4, 4), 0), ((2, 16, 4, 4), 0),
    ((2, 32, 4, 4), 1), ((2, 64, 4, 8), 1), ((2, 64, 4, 9), 0), ((8, 32, 4, 4), 0), ((1, 32, 4, 4), 0),
    ((4, 32, 1, 32), 1), ((4, 32, 1, 33), 0),
]
WS_OK = [((64, 256), 1), ((128, 256), 1), ((256, 256), 1), ((256, 32), 1), ((32, 256), 0), ((96, 256), 0),
         ((320, 256), 0), ((256, 48), 0), ((256, 0), 0), ((0, 256), 0)]

UNSIZED = {"msda_abi_version", "msda_strerror", "msda_uses_fast_path", "msda_launch_count", "msda_set_knob",
           "msda_linear_tf32_ws_ok"}


@pytest.fixture(scope="module")
def lib():
    from uninext_b200 import _cabi, build
    return _cabi.load(build.build())


def _limit_ids():
    return [(fn, i) for fn, spec in sorted(SPECS.items()) for i in range(len(spec.limits))]


def test_every_declared_function_has_a_case():
    from uninext_b200 import _cabi
    assert set(_cabi.SIGNATURES) == set(SPECS) | UNSIZED


@pytest.mark.parametrize("fn", sorted(SPECS))
def test_valid_call_gets_past_the_checks(lib, fn):
    spec = SPECS[fn]
    assert spec.call(lib, fn) not in (BADARG, TOOLARGE)
    for over in spec.early:
        assert spec.call(lib, fn, **over) == 0, over


@pytest.mark.parametrize("fn", sorted(SPECS))
def test_null_pointer_is_badarg(lib, fn):
    spec = SPECS[fn]
    for name in spec.ptrs:
        got = spec.call(lib, fn, null=name)
        if name in spec.optional:
            assert got != BADARG, f"{fn}: {name} may be NULL"
        else:
            assert got == BADARG, f"{fn}: {name} NULL"


@pytest.mark.parametrize("fn,i", _limit_ids())
def test_limit(lib, fn, i):
    spec = SPECS[fn]
    over, want = spec.limits[i]
    got = spec.call(lib, fn, **over)
    if want == 0:                               # just inside the limit: gets past the checks
        assert got not in (BADARG, TOOLARGE), over
    else:
        assert got == want, over


def test_optional_pointers(lib):
    p = {n: BASE + (i << 20) for i, n in enumerate(("a", "b", "z", "g", "bt", "y", "mu", "rs", "w", "ws", "pos", "bo",
                                                     "ch"))}
    ln = lib.msda_add_layernorm_forward_f32
    assert ln(p["a"], p["b"], p["g"], p["bt"], 10, 256, 1e-5, None, p["y"], p["mu"], p["rs"], None) == BADARG  # b needs z
    assert ln(p["a"], None, p["g"], p["bt"], 10, 256, 1e-5, None, p["y"], p["mu"], p["rs"], None) not in (BADARG, TOOLARGE)
    enc = lib.msda_mask_rle_encode                                                   # positions may be NULL when B = 0
    assert enc(3, 30, 50, 0, p["ws"], BIG_WS, None, p["bo"], p["ch"], None) not in (BADARG, TOOLARGE)
    assert enc(3, 30, 50, 1, p["ws"], BIG_WS, None, p["bo"], p["ch"], None) == BADARG
    assert enc(3, 30, 50, 1, p["ws"], BIG_WS, p["pos"] + 2, p["bo"], p["ch"], None) == BADARG   # uint32 positions
    assert enc(3, 30, 50, 1, p["ws"], BIG_WS, p["pos"], p["bo"] + 4, p["ch"], None) == BADARG   # int64 offsets
    spec = _vlf_fwd                                                                  # seed is read only when p > 0
    assert spec.call(lib, "msda_vlfuse_forward_f32", null="seed", p=0.0) not in (BADARG, TOOLARGE)
    assert _vlf_bwd.call(lib, "msda_vlfuse_backward_f32", null="seed", p=0.0) not in (BADARG, TOOLARGE)


def test_knobs_and_version(lib):
    assert lib.msda_abi_version() == 11
    for code in (0, BADARG, TOOLARGE, -3, 1, -99):
        assert lib.msda_strerror(code)
    for k in (-1, 10, 1000):
        assert lib.msda_set_knob(k, 0) == BADARG
    defaults = {0: -1, 1: -1, 2: 48, 3: 2, 4: 0, 5: 0, 6: 0, 7: 0, 8: 2, 9: -1}
    import os
    for k, v in defaults.items():
        env = ["SLAB", "BWD_WIN_ROWS", "BWD_LIST_CAP", "FWD_SLAB_CTAS", "F32_VEC8_FWD", "F32_VEC8_BWD",
               "BF16_FINE_ROWS", "BF16_PACKED_FWD", "ZERO_FILL", "REGION_BWD"][k]
        if not os.environ.get("MSDA_" + env):
            assert lib.msda_set_knob(k, -1000000) == v, env


@pytest.mark.parametrize("args,want", FAST_PATH)
def test_uses_fast_path(lib, args, want):
    assert lib.msda_uses_fast_path(*args) == want


@pytest.mark.parametrize("args,want", WS_OK)
def test_linear_ws_ok(lib, args, want):
    assert lib.msda_linear_tf32_ws_ok(*args) == want


@pytest.mark.parametrize("fn,sizes,want", WORKSPACE)
def test_workspace_bytes(lib, fn, sizes, want):
    out = ctypes.c_int64(-7)
    assert getattr(lib, fn)(*sizes, ctypes.byref(out)) == 0
    assert out.value == want
