"""The host-side argument checks of the 20 rasterizer entry points (dgr_forward{,_aux,_nrm,_surf},
dgr_backward{,_aux,_cam,_nrm,_surf,_abs} and their _batch forms), without a GPU.

Each row of the table below is one defect in an otherwise well-formed call: a negative or zero size, no frame, too
many frames, a NULL required pointer, near >= far, a missing or short normal / surface / camera-gradient workspace, an
unaligned batch stride.  Every entry point that takes the row's arguments must refuse the call with the row's code
and say so in dgm_last_error().  The pointers are never dereferenced: every row is refused before any device work
(no row has P = 0, whose forward and camera-gradient backward zero their outputs before returning)."""
import ctypes
import os
import re

import pytest

FAKE = 1 << 20
BIG = 1 << 30                          # a workspace size / stride that is large enough and a multiple of 128
TAN = (ctypes.c_float * 128)(*([1.0] * 128))
SINGLE = ["dgr_forward", "dgr_forward_aux", "dgr_forward_nrm", "dgr_forward_surf", "dgr_backward",
          "dgr_backward_aux", "dgr_backward_cam", "dgr_backward_nrm", "dgr_backward_surf", "dgr_backward_abs"]
ENTRIES = SINGLE + [n.replace("_forward", "_forward_batch").replace("_backward", "_backward_batch") for n in SINGLE]


def _header_params(name):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    txt = open(os.path.join(root, "include", "dgmesh_b200.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    decl = re.search(r"\bint\s+" + name + r"\s*\(([^)]*)\)", txt).group(1)
    return {re.split(r"[\s*]+", a.strip())[-1]: "*" in a for a in decl.split(",")}  # name: is a pointer


# a well-formed call: colours precomputed, scales + rotations, every optional map and gradient absent
BASE = dict(F=2, P=10, D=0, M=0, W=64, H=48, R_cap=4096, scale_modifier=1.0, tan_fovx=1.0, tan_fovy=1.0,
            tan_fovx_host=TAN, tan_fovy_host=TAN, near=0.5, far=20.0, n_streams=1,
            geom_bytes=BIG, binning_bytes=BIG, img_bytes=BIG, geom_stride=BIG, binning_stride=BIG, img_stride=BIG)
for _p in ("background", "means3D", "colors_precomp", "opacities", "scales", "rotations", "viewmatrix", "projmatrix",
           "cam_pos", "viewmatrices", "projmatrices", "cam_poses", "out_color", "radii", "geom_ws", "binning_ws",
           "img_ws", "status", "dL_dpix", "dL_dmean2D", "dL_dconic", "dL_dopacity", "dL_dcolor", "dL_dmean3D",
           "dL_dcov3D", "dL_dscale", "dL_drot"):
    BASE[_p] = FAKE
NRM_FWD = dict(normals=FAKE, out_normal=FAKE, nrm_ws=FAKE, nrm_ws_bytes=BIG, nrm_ws_stride=BIG)
SURF_FWD = dict(out_median=FAKE, surf_ws=FAKE, surf_ws_bytes=BIG, surf_ws_stride=BIG)
CAM_BWD = dict(dL_dviewmatrix=FAKE, dL_dviewmatrices=FAKE, cam_ws=FAKE, cam_ws_bytes=BIG)
NRM_BWD = dict(dL_dnormal_map=FAKE, dL_dnormal_maps=FAKE, nrm_ws=FAKE, nrm_ws_stride=BIG)
SURF_BWD = dict(dL_dmedian=FAKE, surf_ws=FAKE, surf_ws_stride=BIG)


def _null(*names):
    return [dict.fromkeys([n], None) for n in names]


# (entry points: "fwd" / "bwd" x "one" / "batch", the arguments that differ from BASE, code, text of the message)
ROWS = [
    ("fwd bwd one batch", dict(P=-1), -1, b"size"),
    ("fwd bwd one batch", dict(W=0), -1, b"size"),
    ("fwd bwd one batch", dict(H=-4), -1, b"size"),
    ("fwd bwd one batch", dict(R_cap=-1), -1, b"size"),
    ("fwd batch", dict(F=0), -1, b"bad argument"),
    ("bwd batch", dict(F=0), -1, b"bad size"),
    ("bwd batch", dict(F=65), -1, b"64 frames"),
]
ROWS += [("fwd one", o, -1, b"null required pointer")
         for o in _null("background", "viewmatrix", "projmatrix", "cam_pos", "out_color", "status")]
ROWS += [("fwd batch", o, -1, b"bad argument")
         for o in _null("viewmatrices", "projmatrices", "cam_poses", "tan_fovx_host", "tan_fovy_host")]
ROWS += [("fwd batch", o, -1, b"null required pointer") for o in _null("background", "out_color", "status")]
ROWS += [("fwd one batch", o, -1, b"means3D / opacities") for o in _null("means3D", "opacities")]
ROWS += [
    ("fwd one batch", dict(colors_precomp=None), -1, b"exactly one of shs / colors_precomp"),
    ("fwd one batch", dict(shs=FAKE), -1, b"exactly one of shs / colors_precomp"),
    ("fwd one batch", dict(scales=None), -1, b"exactly one of scales+rotations"),
    ("fwd one batch", dict(cov3D_precomp=FAKE), -1, b"exactly one of scales+rotations"),
    ("fwd one batch", dict(shs=FAKE, colors_precomp=None, D=1, M=3), -1, b"SH degree"),
    ("fwd one batch", dict(shs=FAKE, colors_precomp=None, D=0, M=17), -1, b"SH degree"),
]
ROWS += [("fwd one", o, -2, b"workspace too small") for o in _null("geom_ws", "binning_ws", "img_ws")]
ROWS += [("fwd one", {k: 1000}, -2, b"workspace too small") for k in ("geom_bytes", "binning_bytes", "img_bytes")]
ROWS += [("fwd batch", {k: s}, -2, b"stride") for k in ("geom_stride", "binning_stride", "img_stride")
         for s in (1024, BIG + 64)]
ROWS += [
    ("fwd one batch nrm", dict(NRM_FWD, normals=None), -1, b"normals missing"),
    ("fwd one batch nrm", dict(NRM_FWD, nrm_ws=None), -2, b"normal workspace"),
    ("fwd one nrm", dict(NRM_FWD, nrm_ws_bytes=64), -2, b"normal workspace"),
    ("fwd batch nrm", dict(NRM_FWD, nrm_ws_stride=64), -2, b"normal workspace"),
    ("fwd batch nrm", dict(NRM_FWD, nrm_ws_stride=BIG + 64), -1, b"stride"),
    ("fwd one batch surf", dict(SURF_FWD, near=0.0), -1, b"near"),
    ("fwd one batch surf", dict(SURF_FWD, near=20.0), -1, b"near"),
    ("fwd one batch surf", dict(SURF_FWD, far=float("inf")), -1, b"near"),
    ("fwd one batch surf", dict(SURF_FWD, out_median=None, out_distortion=FAKE, surf_ws=None), -2,
     b"surface workspace"),
    ("fwd one surf", dict(SURF_FWD, surf_ws_bytes=64), -2, b"surface workspace"),
    ("fwd batch surf", dict(SURF_FWD, surf_ws_stride=64), -2, b"surface workspace"),
    ("fwd batch surf", dict(SURF_FWD, surf_ws_stride=BIG + 64), -1, b"stride"),
]
ROWS += [("bwd one", o, -1, b"null required pointer")
         for o in _null("background", "means3D", "viewmatrix", "projmatrix", "cam_pos", "geom_ws", "binning_ws",
                        "img_ws", "dL_dpix", "dL_dmean2D", "dL_dopacity", "dL_dcolor", "dL_dmean3D", "dL_dcov3D",
                        "dL_dscale", "dL_drot")]
ROWS += [("bwd batch", o, -1, b"null required pointer")
         for o in _null("background", "means3D", "viewmatrices", "projmatrices", "cam_poses", "tan_fovx_host",
                        "tan_fovy_host", "geom_ws", "binning_ws", "img_ws", "dL_dpix", "dL_dmean2D", "dL_dopacity",
                        "dL_dcolor", "dL_dmean3D", "dL_dscale", "dL_drot")]
ROWS += [
    ("bwd batch", dict(cov3D_precomp=FAKE, dL_dcov3D=None), -1, b"null required pointer"),
    ("bwd batch", dict(shs=FAKE, colors_precomp=None), -1, b"null required pointer"),
    ("bwd one", dict(shs=FAKE, colors_precomp=None), -1, b"dL_dsh missing"),
    ("bwd one batch cam", dict(CAM_BWD, cam_ws=None), -2, b"camera-gradient workspace"),
    ("bwd one batch cam", dict(CAM_BWD, cam_ws_bytes=64), -2, b"camera-gradient workspace"),
    ("bwd one batch cam", dict(CAM_BWD, dL_dviewmatrix=None, dL_dviewmatrices=None, dL_dcampos=FAKE,
                               dL_dcam_poses=FAKE, cam_ws_bytes=0), -2, b"camera-gradient workspace"),
    ("bwd one batch nrm", dict(NRM_BWD, nrm_ws=None), -1, b"normal workspace missing"),
    ("bwd batch nrm", dict(NRM_BWD, nrm_ws_stride=BIG + 64), -1, b"stride"),
    ("bwd one batch surf", dict(SURF_BWD, near=-1.0), -1, b"near"),
    ("bwd one batch surf", dict(SURF_BWD, far=0.25), -1, b"near"),
    ("bwd one batch surf", dict(SURF_BWD, dL_dmedian=None, dL_ddistortion=FAKE, surf_ws=None), -1,
     b"surface workspace missing"),
    ("bwd batch surf", dict(SURF_BWD, surf_ws_stride=BIG + 64), -1, b"stride"),
    ("bwd batch surf", dict(SURF_BWD, surf_ws_stride=1024), -1, b"stride"),
]
# the batch forward with several streams takes another schedule; its checks are the same
ROWS += [(kinds, dict(o, n_streams=4), rc, text) for kinds, o, rc, text in list(ROWS)
         if kinds.startswith("fwd") and "batch" in kinds and not set(o) & {"means3D", "opacities"}]


# a row on the normal map, the surface maps or the camera gradients applies to the entry points with that argument
SEGMENT = {"nrm": "nrm_ws", "surf": "near", "cam": "cam_ws"}


def _cases():
    for kinds, over, rc, text in ROWS:
        kinds = set(kinds.split())
        for name in ENTRIES:
            params = _header_params(name)
            if ("fwd" if "_forward" in name else "bwd") not in kinds:
                continue
            if ("batch" if "_batch" in name else "one") not in kinds:
                continue
            if any(SEGMENT[k] not in params for k in kinds & set(SEGMENT)):
                continue
            shown = ",".join(f"{k}={'NULL' if v is None else v}" for k, v in over.items() if k in params)
            yield pytest.param(name, over, rc, text, id=f"{name}-{shown}")


@pytest.mark.parametrize("name,over,rc,text", list(_cases()))
def test_bad_argument_is_refused_on_the_host(name, over, rc, text):
    import _dgm_lib
    lib = _dgm_lib.lib()
    params = _header_params(name)
    args = dict(BASE, **over)
    # the arguments BASE and the row leave out: NULL pointers and zero numbers
    assert getattr(lib, name)(*[args.get(p, None if ptr else 0) for p, ptr in params.items()]) == rc
    assert text in lib.dgm_last_error(), lib.dgm_last_error()


def test_every_entry_point_is_covered():
    names = {c.values[0] for c in _cases()}
    assert names == set(ENTRIES)
