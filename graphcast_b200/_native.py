"""ctypes binding of libgraphcast_b200.so (the C ABI in include/graphcast_b200.h).

There is NO fallback: if the shared library is missing or does not export the
ABI, importing the product path raises.  Build it with
`graphcast_b200/csrc/build.sh` or `__graft_entry__.build()`.
"""

from __future__ import annotations

import ctypes as C
import os

# GCB_LIB: an alternative build of the same library (kernel experiments); default = the in-tree one.
_LIB_PATH = os.environ.get("GCB_LIB") or os.path.join(os.path.dirname(os.path.abspath(__file__)),
                                                      "libgraphcast_b200.so")

GCB_ABI_VERSION = 2
GCB_MAX_MSG_STEPS = 64
PREC_BF16X3, PREC_BF16, PREC_FP32_SIMT = 0, 1, 2
PRECISIONS = {"bf16x3": PREC_BF16X3, "bf16": PREC_BF16, "fp32_simt": PREC_FP32_SIMT}
ACT_NONE, ACT_SWISH = 0, 1

_fp = C.c_void_p   # device pointers are passed as raw addresses


class Segment(C.Structure):
  _fields_ = [("table", _fp), ("idx", _fp), ("ld", C.c_int32), ("k", C.c_int32),
              ("k_valid", C.c_int32), ("fan", C.c_int32), ("img", _fp)]


class PreAdd(C.Structure):
  _fields_ = [("table", _fp), ("idx", _fp), ("ld", C.c_int32), ("pad_", C.c_int32)]


class LayerDesc(C.Structure):
  _fields_ = [("rows", C.c_int32), ("n", C.c_int32), ("n_valid", C.c_int32),
              ("nseg", C.c_int32), ("seg", Segment * 3),
              ("w_packed", _fp), ("w_f32", _fp), ("bias", _fp),
              ("ln_scale", _fp), ("ln_offset", _fp), ("act", C.c_int32),
              ("residual", _fp), ("ld_res", C.c_int32),
              ("out", _fp), ("ld_out", C.c_int32),
              ("out_y", _fp), ("ld_out_y", C.c_int32),
              ("precision", C.c_int32), ("n_pre_add", C.c_int32), ("pre_add", PreAdd * 2),
              ("out_img", _fp)]


class MlpSplit(C.Structure):
  _fields_ = [("we_packed", _fp), ("we_f32", _fp), ("ws_packed", _fp), ("ws_f32", _fp),
              ("wr_packed", _fp), ("wr_f32", _fp)]


class Mlp(C.Structure):
  _fields_ = [("w0_packed", _fp), ("w0_f32", _fp), ("b0", _fp),
              ("w1_packed", _fp), ("w1_f32", _fp), ("b1", _fp),
              ("ln_scale", _fp), ("ln_offset", _fp),
              ("k0", C.c_int32), ("n1", C.c_int32), ("n1_valid", C.c_int32)]


class Model(C.Structure):
  _fields_ = [
      ("num_grid", C.c_int32), ("num_mesh", C.c_int32),
      ("e_g2m", C.c_int32), ("e_mesh", C.c_int32), ("e_m2g", C.c_int32),
      ("c_in_pad", C.c_int32), ("c_in_valid", C.c_int32),
      ("msg_steps", C.c_int32), ("precision", C.c_int32), ("pregather", C.c_int32),
      ("g2m_snd", _fp), ("g2m_rcv", _fp), ("g2m_row_ptr", _fp), ("g2m_feat", _fp),
      ("g2m_heavy", _fp), ("n_g2m_heavy", C.c_int32),
      ("mesh_snd", _fp), ("mesh_rcv", _fp), ("mesh_row_ptr", _fp), ("mesh_feat", _fp),
      ("m2g_snd", _fp), ("m2g_rcv", _fp), ("m2g_feat", _fp),
      ("mesh_in", _fp),
      ("enc_grid", Mlp), ("enc_mesh", Mlp), ("enc_e_g2m", Mlp), ("proc_e_g2m", Mlp),
      ("proc_n_mesh_g2m", Mlp), ("proc_n_grid_g2m", Mlp),
      ("enc_e_mesh", Mlp),
      ("proc_e_mesh", Mlp * GCB_MAX_MSG_STEPS),
      ("proc_n_mesh", Mlp * GCB_MAX_MSG_STEPS),
      ("enc_e_m2g", Mlp), ("proc_e_m2g", Mlp), ("proc_n_grid_m2g", Mlp), ("dec_grid", Mlp),
      ("proc_e_g2m_split", MlpSplit), ("proc_e_m2g_split", MlpSplit),
      ("proc_e_mesh_split", MlpSplit * GCB_MAX_MSG_STEPS),
      ("zero_bias", _fp), ("proj_grid", _fp), ("proj_mesh_a", _fp), ("proj_mesh_b", _fp),
      ("hidden", _fp), ("edge_a_img", _fp), ("edge_b", _fp), ("mesh_in_img", _fp), ("grid_lat", _fp), ("grid_lat_img", _fp), ("mesh_lat", _fp),
      ("mesh_lat_img", _fp), ("mesh_agg", _fp), ("mesh_agg_img", _fp), ("mesh_edge", _fp),
      ("mesh_edge_img", _fp), ("mesh_msg", _fp), ("grid_agg_img", _fp),
      ("fuse", C.c_int32), ("chain_lag", C.c_int32),
      ("num_grid_owned", C.c_int32), ("num_mesh_owned", C.c_int32),
      ("chain_scratch", _fp),
      ("image_residual", C.c_int32), ("deep_chains", C.c_int32), ("proj_grid_b", _fp),
      ("chain_scratch_bytes", C.c_int64),
  ]


GCB_MAX_CHAIN = 6
STAGE_ENCODE, STAGE_PROCESS_EMBED, STAGE_PROCESS_STEP, STAGE_DECODE = 0, 1, 2, 3


class ChainLayer(C.Structure):
  _fields_ = [("nseg", C.c_int32), ("seg", Segment * 3), ("seg_from", C.c_int32 * 3),
              ("w_packed", _fp), ("bias", _fp), ("ln_scale", _fp), ("ln_offset", _fp),
              ("act", C.c_int32), ("keep", C.c_int32),
              ("residual", _fp), ("ld_res", C.c_int32),
              ("residual_img", _fp), ("residual_keep", C.c_int32),
              ("out", _fp), ("ld_out", C.c_int32),
              ("out_y", _fp), ("ld_out_y", C.c_int32),
              ("out_img", _fp),
              ("n_pre_add", C.c_int32), ("pre_add", PreAdd * 2)]


class ChainDesc(C.Structure):
  _fields_ = [("rows", C.c_int32), ("nlayers", C.c_int32), ("precision", C.c_int32),
              ("lag", C.c_int32), ("order", C.c_int32), ("pad_", C.c_int32), ("scratch", _fp),
              ("scratch_bytes", C.c_int64), ("layer", ChainLayer * GCB_MAX_CHAIN)]


# name -> (restype, argtypes); every symbol declared in include/graphcast_b200.h.
EXPORTS = {
    "gcb_abi_version": (C.c_int, []),
    "gcb_last_error": (C.c_char_p, []),
    "gcb_sm_count": (C.c_int, [C.c_int]),
    "gcb_packed_weight_bytes": (C.c_int64, [C.c_int32, C.c_int32]),
    "gcb_a_image_bytes": (C.c_int64, [C.c_int64, C.c_int32]),
    "gcb_rows_to_image": (C.c_int, [_fp, C.c_int32, C.c_int32, C.c_int64, C.c_int32, _fp, _fp]),
    "gcb_gather_rows": (C.c_int, [_fp, C.c_int32, _fp, C.c_int64, _fp, C.c_int32, C.c_int32, _fp]),
    "gcb_image_rows_pack": (C.c_int, [_fp, _fp, C.c_int64, _fp, _fp]),
    "gcb_image_rows_unpack": (C.c_int, [_fp, C.c_int64, _fp, C.c_int64, _fp]),
    "gcb_pack_weight_host": (C.c_int, [_fp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _fp]),
    "gcb_pack_weight": (C.c_int, [_fp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                  C.c_int32, _fp, _fp, _fp]),
    "gcb_sum_squares": (C.c_int, [_fp, C.c_int64, _fp, C.c_int64, _fp, _fp]),
    "gcb_sum_squares_workspace_bytes": (C.c_int64, []),
    "gcb_adamw_step": (C.c_int, [_fp, _fp, _fp, _fp, C.c_int64, C.c_int64, C.c_int64, C.c_double,
                                 C.c_double, C.c_double, C.c_double, C.c_double, C.c_double, _fp,
                                 C.c_double, _fp]),
    "gcb_layer_forward": (C.c_int, [C.POINTER(LayerDesc), _fp]),
    "gcb_segment_sum": (C.c_int, [_fp, C.c_int32, _fp, C.c_int32, _fp, C.c_int32, C.c_int32, _fp]),
    "gcb_segment_sum_heavy": (C.c_int, [_fp, C.c_int32, _fp, C.c_int32, _fp, C.c_int32, _fp,
                                        C.c_int32, C.c_int32, _fp]),
    "gcb_pack_grid_features": (C.c_int, [_fp, C.c_int32, C.c_int64, _fp, _fp, _fp, C.c_int32,
                                         _fp, C.c_int32, _fp]),
    "gcb_pack_grid_image": (C.c_int, [_fp, C.c_int32, C.c_int64, _fp, _fp, _fp, C.c_int32,
                                      C.c_int32, _fp, _fp]),
    "gcb_unpack_grid_outputs": (C.c_int, [_fp, C.c_int32, C.c_int32, C.c_int64, _fp, _fp, _fp,
                                          _fp, _fp, _fp]),
    "gcb_output_loss": (C.c_int, [_fp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _fp, _fp, _fp,
                                  _fp, _fp, _fp, _fp, _fp, C.c_int64, _fp, _fp]),
    "gcb_output_loss_workspace_bytes": (C.c_int64, [C.c_int32]),
    "gcb_output_loss_grad": (C.c_int, [_fp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _fp, _fp,
                                       _fp, _fp, _fp, _fp, _fp, _fp, C.c_int32, _fp]),
    "gcb_output_loss_grad_feedback": (C.c_int, [_fp, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                                _fp, _fp, _fp, _fp, _fp, _fp, _fp, _fp, _fp,
                                                C.c_int32, _fp, _fp, _fp, _fp, C.c_int32, _fp]),
    "gcb_input_grad": (C.c_int, [_fp, C.c_int32, C.c_int64, C.c_int32, _fp, _fp, _fp, C.c_int32,
                                 _fp]),
    "gcb_weight_grad_workspace_bytes": (C.c_int64, [C.c_int32, C.c_int32]),
    "gcb_weight_grad": (C.c_int, [_fp, C.c_int32, C.c_int32, _fp, C.c_int32, _fp, C.c_int32,
                                  C.c_int64, C.c_int32, C.c_int32, C.c_int32, _fp, C.c_int64, _fp,
                                  C.c_int32, _fp]),
    "gcb_rowwise_workspace_bytes": (C.c_int64, [C.c_int32]),
    "gcb_layernorm_backward": (C.c_int, [_fp, C.c_int32, _fp, C.c_int32, _fp, C.c_int64, C.c_int32,
                                         _fp, C.c_int32, _fp, C.c_int64, _fp, _fp, _fp, C.c_int32,
                                         _fp]),
    "gcb_swish_backward": (C.c_int, [_fp, C.c_int32, _fp, C.c_int32, C.c_int64, C.c_int32, _fp,
                                     C.c_int32, _fp, C.c_int64, _fp, C.c_int32, _fp]),
    "gcb_segment_sum_sorted": (C.c_int, [_fp, C.c_int32, _fp, _fp, C.c_int32, _fp, C.c_int32, _fp,
                                         C.c_int32, C.c_int32, _fp]),
    "gcb_swish_rows": (C.c_int, [_fp, C.c_int32, C.c_int64, C.c_int32, _fp, C.c_int32, _fp]),
    "gcb_gather_add": (C.c_int, [_fp, C.c_int32, _fp, C.c_int64, _fp, C.c_int32, _fp, C.c_int32,
                                 C.c_int32, _fp]),
    "gcb_forward":(C.c_int, [C.POINTER(Model), _fp, _fp, _fp, C.POINTER(C.c_int32)]),
    "gcb_forward_stage": (C.c_int, [C.POINTER(Model), C.c_int32, C.c_int32, _fp, _fp, _fp,
                                    C.POINTER(C.c_int32)]),
    "gcb_chain_scratch_bytes": (C.c_int64, [C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    "gcb_chain_forward": (C.c_int, [C.POINTER(ChainDesc), _fp]),
    "gcb_set_cluster_size": (C.c_int, [C.c_int32]),
    "gcb_toa_incident_solar_radiation": (C.c_int, [_fp, C.c_int32, C.c_int32, _fp, _fp, _fp, _fp,
                                         C.c_int32, C.c_int32, _fp, _fp]),
    "gcb_set_graph_replay": (C.c_int, [C.c_int32]),
    "gcb_debug_trace": (C.c_int, [_fp]),
    "gcb_debug_flags": (C.c_int, [C.c_int]),
    "gcb_profile_begin": (C.c_int, []),
    "gcb_profile_end": (C.c_int, [C.c_int32, _fp, _fp, _fp, _fp, C.POINTER(C.c_int32)]),
    "gcb_selftest_layer": (C.c_int, [C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                     C.POINTER(C.c_float)]),
}


class NativeLibraryError(RuntimeError):
  pass


_lib = None


def lib():
  """Loads the shared library once; raises NativeLibraryError if unavailable."""
  global _lib
  if _lib is not None:
    return _lib
  if not os.path.exists(_LIB_PATH):
    raise NativeLibraryError(
        f"{_LIB_PATH} not found: build it with graphcast_b200/csrc/build.sh "
        "(there is no CPU / PyTorch fallback for the GraphCast hot path)")
  try:
    handle = C.CDLL(_LIB_PATH)
  except OSError as e:
    raise NativeLibraryError(f"cannot load {_LIB_PATH}: {e}") from e
  for name, (restype, argtypes) in EXPORTS.items():
    try:
      fn = getattr(handle, name)
    except AttributeError as e:
      raise NativeLibraryError(f"{_LIB_PATH} does not export {name}") from e
    fn.restype = restype
    fn.argtypes = argtypes
  if handle.gcb_abi_version() != GCB_ABI_VERSION:
    raise NativeLibraryError("ABI version mismatch between _native.py and the library")
  if os.environ.get("GCB_NO_GRAPH"):      # debugging aid: plain launches instead of graph replay
    handle.gcb_set_graph_replay(0)
  _lib = handle
  return _lib


def check(rc: int, what: str = "") -> None:
  if rc != 0:
    msg = lib().gcb_last_error().decode("utf-8", "replace")
    if rc == -1:
      raise ValueError(f"{what}: {msg}")
    raise RuntimeError(f"{what}: gcb status {rc}: {msg}")
