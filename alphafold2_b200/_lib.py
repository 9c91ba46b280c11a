"""ctypes binding of libaf2b200.so (include/af2b200.h).  No torch extension, no pybind: the C ABI is the
drop-in boundary.  There is deliberately NO fallback: if the library is missing or the device is not
sm_90 (H100), every op raises."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# AF2_LIB_PATH: A/B builds of the same library on one machine; never a different implementation
LIB_PATH = os.environ.get("AF2_LIB_PATH") or os.path.join(_HERE, "csrc", "libaf2b200.so")

_lib = None

vp, ll, ci, cf = C.c_void_p, C.c_longlong, C.c_int, C.c_float


class FFWeights(C.Structure):
    _fields_ = [("ln_gamma", vp), ("ln_beta", vp), ("w1", vp), ("b1", vp), ("w2", vp), ("b2", vp), ("bn", ci)]


class AttnWeights(C.Structure):
    _fields_ = [("ln_gamma", vp), ("ln_beta", vp), ("w_qkv", vp), ("w_gate", vp), ("b_gate", vp),
                ("w_out", vp), ("b_out", vp), ("w_edge", vp)]


class TriMulWeights(C.Structure):
    _fields_ = [("ln_gamma", vp), ("ln_beta", vp), ("w_left", vp), ("b_left", vp), ("w_right", vp),
                ("b_right", vp), ("w_ogate", vp), ("b_ogate", vp), ("on_gamma", vp), ("on_beta", vp),
                ("w_out", vp), ("b_out", vp), ("bn", ci)]


class OuterWeights(C.Structure):
    _fields_ = [("ln_gamma", vp), ("ln_beta", vp), ("w_lr", vp), ("b_lr", vp), ("w_out", vp), ("b_out", vp)]


class GemmEpilogue(C.Structure):
    _fields_ = [("bn", ci), ("mode", ci), ("act", ci), ("layout", ci), ("use_rowscale", ci), ("bias", vp), ("rowscale", vp),
                ("resid", vp), ("ld_resid", ll), ("out", vp), ("ld_out", ll), ("out_batch", ll), ("cm_inner", ci),
                ("cm_pitch", ci), ("out_cols", ci)]


class FFWeightsStrict(C.Structure):
    _fields_ = [("ln_gamma", vp), ("ln_beta", vp), ("w1", vp), ("b1", vp), ("w2", vp), ("b2", vp)]


class AttnWeightsStrict(C.Structure):
    _fields_ = [("ln_gamma", vp), ("ln_beta", vp), ("w_qkvg", vp), ("b_qkvg", vp), ("w_out", vp), ("b_out", vp), ("w_edge", vp)]


class TriMulWeightsStrict(C.Structure):
    _fields_ = [("ln_gamma", vp), ("ln_beta", vp), ("w5", vp), ("b5", vp), ("on_gamma", vp), ("on_beta", vp),
                ("w_out", vp), ("b_out", vp)]


class OuterWeightsStrict(C.Structure):
    _fields_ = [("ln_gamma", vp), ("ln_beta", vp), ("w_lr", vp), ("b_lr", vp), ("w_out", vp), ("b_out", vp)]


class TemplateAttnWeights(C.Structure):
    _fields_ = [("w_q", vp), ("w_gate", vp), ("b_gate", vp), ("w_kv", vp), ("w_out", vp), ("b_out", vp)]


class TemplateAttnWeightsStrict(C.Structure):
    _fields_ = [("w_qg", vp), ("b_qg", vp), ("w_kv", vp), ("w_out", vp), ("b_out", vp)]


class TemplateAngleWeights(C.Structure):
    _fields_ = [("w1", vp), ("b1", vp), ("w2", vp), ("b2", vp)]


TemplateAngleWeightsStrict = TemplateAngleWeights      # same layout, split-bf16 weights


class StructureWeights(C.Structure):
    _fields_ = [(k, vp) for k in ("w_proj", "w_bias", "b_bias", "point_weights", "w_out", "b_out", "attn_gamma", "attn_beta", "w_ff0",
                                  "b_ff0", "w_ff2", "b_ff2", "w_ff4", "b_ff4", "ff_gamma", "ff_beta", "w_qu", "b_qu", "w_points",
                                  "b_points", "w_lddt", "b_lddt")]


class Points(C.Structure):
    """af2_points: coordinate k of point i of element e at p[e * sb + i * sn + k * sk]."""
    _fields_ = [("p", vp), ("sb", ll), ("sn", ll), ("sk", ll)]


class GdtSpec(C.Structure):
    _fields_ = [("out", vp), ("k", ci), ("idx", ci * 8), ("w", cf * 8)]


class PeerChunk(C.Structure):
    _fields_ = [("src_off", ll), ("dst_off", ll), ("dst_row_stride", ll), ("row_bytes", ll), ("rows", ci), ("reserved", ci)]


_SIGNATURES = {
    "af2_last_error": (C.c_char_p, []),
    "af2_abi_version": (ci, []),
    "af2_check_device": (ci, []),
    "af2_launch_count": (C.c_ulonglong, []),
    "af2_profile_enable": (None, [ci]),
    "af2_profile_read": (ll, [ci, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double)]),
    "af2_feed_forward": (ci, [C.POINTER(FFWeights), vp, ll, ci, ci, vp, ll, vp]),
    "af2_feed_forward_workspace": (ll, [ll, ci, ci]),
    "af2_axial_attention": (ci, [C.POINTER(AttnWeights), vp, vp, vp, ci, ci, ci, ci, ci, ci, ci, vp, ll, vp]),
    "af2_axial_attention_ex": (ci, [C.POINTER(AttnWeights), vp, vp, vp, ci, ci, ci, ci, ci, ci, ci, ci, vp, ll, vp]),
    "af2_axial_attention_workspace": (ll, [ci, ci, ci, ci, ci, ci, ci]),
    "af2_triangle_multiply": (ci, [C.POINTER(TriMulWeights), vp, vp, ci, ci, ci, ci, vp, ll, vp]),
    "af2_triangle_multiply_workspace": (ll, [ci, ci, ci]),
    "af2_outer_mean": (ci, [C.POINTER(OuterWeights), vp, vp, vp, ci, ci, ci, ci, cf, vp, ll, vp]),
    "af2_outer_mean_workspace": (ll, [ci, ci, ci, ci]),
    "af2_pair_bias": (ci, [vp, vp, vp, ci, ci, ci, ci, vp]),
    "af2_axial_attention_prebias": (ci, [C.POINTER(AttnWeights), vp, vp, vp, ci, ci, ci, ci, ci, ci, ci, vp, ll, vp]),
    "af2_axial_attention_tied_begin": (ci, [C.POINTER(AttnWeights), vp, vp, vp, ci, ci, ci, ci, ci, vp, vp, ll, vp]),
    "af2_axial_attention_tied_end": (ci, [C.POINTER(AttnWeights), vp, vp, vp, ci, ci, ci, ci, ci, vp, ci, ci, vp, ll, vp]),
    "af2_triangle_project": (ci, [C.POINTER(TriMulWeights), vp, vp, ll, ci, ci, vp, vp, ll, vp, vp, ll, vp]),
    "af2_triangle_project_workspace": (ll, [ll, ci]),
    "af2_triangle_contract": (ci, [C.POINTER(TriMulWeights), vp, vp, ll, ll, vp, ll, ll, ll, ci, vp, ci, ci, ci, ci, ci, vp, ll, vp]),
    "af2_triangle_contract_workspace": (ll, [ci, ci, ci]),
    "af2_outer_project": (ci, [C.POINTER(OuterWeights), vp, vp, ll, ci, ci, vp, ll, vp, ll, vp]),
    "af2_outer_project_workspace": (ll, [ll, ci]),
    "af2_outer_contract": (ci, [C.POINTER(OuterWeights), vp, vp, ll, vp, ll, ll, ci, vp, ci, ci, ci, ci, ci, cf, vp, ll, vp]),
    "af2_outer_contract_workspace": (ll, [ci, ci, ci]),
    "af2_rotary": (ci, [vp, vp, vp, vp, ci, ci, ci, ci, ci, ci, vp]),
    "af2_layernorm_bf16": (ci, [vp, vp, vp, vp, ll, ci, cf, vp]),
    "af2_gemm_bf16_f32": (ci, [vp, ll, ll, vp, ll, ll, vp, ll, ll, ci, ci, ci, ci, ci, vp]),
    "af2_gemm_bf16_epilogue": (ci, [vp, ll, ll, vp, ll, ll, ci, ci, ci, ci, ci, C.POINTER(GemmEpilogue), vp]),
    "af2_attention_bf16": (ci, [vp, vp, vp, vp, vp, ci, ci, ci, ci, ll, ll, vp]),
    "af2_attention_proj_bf16": (ci, [vp, ci, vp, vp, vp, vp, vp, vp, ci, ci, ci, ci, ll, ll, vp]),
    "af2_attention_proj_max_n": (ci, [ci]),
    "af2_gemm_bf16_f32_gathered": (ci, [vp, ll, ll, vp, ll, ll, vp, ll, ll, ci, ci, ci, ci, ci, ci, ci, ll, ci, ll, vp]),
    "af2_chan_to_token": (ci, [vp, ll, ci, ci, ci, ci, ci, vp, vp, vp, vp, cf, cf, vp, ci, C.POINTER(ci), vp]),
    "af2_chan_to_token_select": (ci, [vp, ll, ci, ci, ci, ci, ci, vp, vp, vp, vp, cf, cf, vp]),
    "af2_contract_tail": (ci, [vp, ll, ci, ci, ci, ci, ci, vp, vp, vp, vp, cf, cf, vp, vp, vp, vp, vp, vp, vp, ci, C.POINTER(ci), vp]),
    "af2_outer_scale": (ci, [vp, vp, vp, ci, ci, ci, ci, cf, ci, C.POINTER(ci), vp]),
    # strict precision mode (split-bf16 x3 operands)
    "af2_feed_forward_strict": (ci, [C.POINTER(FFWeightsStrict), vp, ll, ci, ci, vp, ll, vp]),
    "af2_feed_forward_strict_workspace": (ll, [ll, ci, ci]),
    "af2_axial_attention_strict": (ci, [C.POINTER(AttnWeightsStrict), vp, vp, vp, ci, ci, ci, ci, ci, ci, ci, ci, vp, ll, vp]),
    "af2_axial_attention_strict_workspace": (ll, [ci, ci, ci, ci, ci, ci, ci]),
    "af2_triangle_multiply_strict": (ci, [C.POINTER(TriMulWeightsStrict), vp, vp, ci, ci, ci, ci, vp, ll, vp]),
    "af2_triangle_multiply_strict_workspace": (ll, [ci, ci, ci]),
    "af2_outer_mean_strict": (ci, [C.POINTER(OuterWeightsStrict), vp, vp, vp, ci, ci, ci, ci, cf, vp, ll, vp]),
    "af2_outer_mean_strict_workspace": (ll, [ci, ci, ci, ci]),
    "af2_embed_pair_init_workspace": (ll, [ci, ci, ci]),
    "af2_embed_pair_init": (ci, [vp, vp, vp, ci, vp, vp, vp, vp, vp, ci, vp, vp, vp, ci, ci, ci, ci, vp, ll, vp]),
    "af2_distogram_head": (ci, [vp, vp, vp, vp, vp, vp, ci, ci, ci, ci, vp]),
    "af2_angle_heads": (ci, [vp, vp, vp, vp, vp, vp, ci, ci, ci, ci, ci, ci, ci, vp]),
    "af2_recycle_embed": (ci, [vp, ci, vp, vp, vp, vp, vp, vp, vp, vp, ci, vp, vp, ll, ci, ci, ci, cf, vp]),
    "af2_embed_pair_init_rows": (ci, [vp, vp, vp, ci, vp, vp, vp, vp, vp, ci, vp, vp, vp, ci, ci, ci, ci, ci, ci, vp, ll, vp]),
    "af2_distogram_head_rows": (ci, [vp, vp, vp, vp, vp, vp, vp, ci, ci, ci, ci, vp]),
    "af2_angle_heads_rows": (ci, [vp, vp, vp, vp, vp, vp, vp, ci, ci, ci, ci, ci, ci, ci, vp]),
    "af2_recycle_embed_rows": (ci, [vp, ci, vp, vp, vp, vp, vp, vp, vp, vp, ci, vp, vp, ll, ci, ci, ci, cf, ci, ci, vp]),
    "af2_split_bf16": (ci, [vp, vp, ll, ci, vp]),
    "af2_gemm_split_f32": (ci, [vp, vp, vp, ll, ci, ci, ci, ci, vp]),
    "af2_gemm_split_epilogue": (ci, [vp, ll, ll, ll, vp, ll, ll, ll, ci, ci, ci, ci, ci, C.POINTER(GemmEpilogue), vp]),
    "af2_strict_ln_split": (ci, [vp, vp, vp, vp, ll, ci, vp]),
    "af2_strict_geglu_split": (ci, [vp, vp, ll, ci, vp]),
    "af2_strict_gelu_split": (ci, [vp, vp, ll, ci, vp]),
    "af2_strict_qkv_split": (ci, [vp, vp, vp, vp, ci, ci, ci, ci, ci, ll, ll, vp]),
    "af2_strict_pair_bias": (ci, [vp, vp, vp, ll, ci, ci, vp]),
    "af2_strict_softmax_split": (ci, [vp, ll, vp, vp, vp, ci, ci, ci, ci, ll, ll, vp]),
    "af2_strict_gate_split": (ci, [vp, ll, vp, vp, ci, ci, ci, ci, ci, ll, ll, vp]),
    "af2_strict_tok2chan_split": (ci, [vp, ll, ci, ci, vp, vp, ci, ci, ci, ll, ll, ll, vp]),
    "af2_strict_chan_to_token": (ci, [vp, ll, ci, ci, ci, ci, ci, vp, vp, vp, ll, ci, vp, cf, cf, vp, vp]),
    "af2_tie_queries_f32": (ci, [vp, ll, ci, ci, ci, ll, ll, vp]),
    "af2_tie_queries_bf16": (ci, [vp, ll, ci, ci, ci, ll, ll, vp]),
    "af2_attention_x_bf16": (ci, [vp, vp, vp, vp, ll, vp, vp, ci, ci, ci, ci, ci, vp, vp]),
    "af2_attn_bias_log2": (ci, [vp, ll, ll, ll, ll, vp, ci, ci, ci, ci, vp]),
    "af2_strict_xqkv_split": (ci, [vp, vp, vp, vp, vp, ci, ci, ci, ci, ci, ci, vp]),
    "af2_strict_xsoftmax_split": (ci, [vp, ll, vp, ll, ll, ll, ll, vp, vp, vp, ci, ci, ci, ci, ci, vp]),
    "af2_strict_xgate_split": (ci, [vp, vp, vp, ci, ci, ci, ci, ci, vp]),
    # template embedder (alphafold2.py:743-792)
    "af2_template_pointwise_attention": (ci, [C.POINTER(TemplateAttnWeights), vp, vp, vp, vp, ci, ci, ci, ci, ci, ci, vp, ll, vp]),
    "af2_template_pointwise_attention_workspace": (ll, [ci, ci, ci, ci, ci, ci]),
    "af2_template_pointwise_attention_strict": (ci, [C.POINTER(TemplateAttnWeightsStrict), vp, vp, vp, vp, ci, ci, ci, ci, ci, ci, vp, ll,
                                                     vp]),
    "af2_template_pointwise_attention_strict_workspace": (ll, [ci, ci, ci, ci, ci, ci]),
    "af2_template_pointwise_bf16_state": (ci, [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, ci, ci, ci, ci, ll, ci, ci, vp]),
    "af2_template_pointwise_f32_state": (ci, [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, ci, ci, ci, ci, ll, ci, ci, vp]),
    "af2_template_pointwise_begin_workspace": (ll, [ll, ci]),
    "af2_template_pointwise_begin": (ci, [C.POINTER(TemplateAttnWeights), vp, ll, ci, ci, ci, vp, vp, vp, ll, vp]),
    "af2_template_pointwise_group_workspace": (ll, [ci, ci, ll, ll, ci, ci, ci]),
    "af2_template_pointwise_group": (ci, [C.POINTER(TemplateAttnWeights), vp, vp, vp, ci, ci, ll, ll, ci, ci, ci, vp, vp, vp, vp, vp,
                                          vp, vp, ci, ci, vp, ll, vp]),
    "af2_template_pointwise_end_workspace": (ll, [ll, ci, ci]),
    "af2_template_pointwise_end": (ci, [C.POINTER(TemplateAttnWeights), vp, vp, vp, ll, ci, ci, ci, vp, ll, vp]),
    "af2_template_pointwise_begin_strict_workspace": (ll, [ll, ci]),
    "af2_template_pointwise_begin_strict": (ci, [C.POINTER(TemplateAttnWeightsStrict), vp, ll, ci, ci, ci, vp, vp, ll, vp]),
    "af2_template_pointwise_group_strict_workspace": (ll, [ci, ci, ll, ll, ci, ci, ci]),
    "af2_template_pointwise_group_strict": (ci, [C.POINTER(TemplateAttnWeightsStrict), vp, vp, vp, ci, ci, ll, ll, ci, ci, ci, vp, vp,
                                                 vp, vp, vp, vp, ci, ci, vp, ll, vp]),
    "af2_template_pointwise_end_strict_workspace": (ll, [ll, ci, ci]),
    "af2_template_pointwise_end_strict": (ci, [C.POINTER(TemplateAttnWeightsStrict), vp, vp, vp, ll, ci, ci, ci, vp, ll, vp]),
    # Attention.forward on its own (alphafold2.py:125-190)
    "af2_attention_forward_workspace": (ll, [ci, ci, ci, ci, ci, ci, ci, ci]),
    "af2_attention_forward": (ci, [C.POINTER(TemplateAttnWeights), vp, vp, vp, vp, vp, ll, ll, ll, ll, ci, ci, ci, ci, ci, ci, ci, vp,
                                   vp, ll, vp]),
    "af2_attention_forward_strict_workspace": (ll, [ci, ci, ci, ci, ci, ci, ci, ci]),
    "af2_attention_forward_strict": (ci, [C.POINTER(TemplateAttnWeightsStrict), vp, vp, vp, vp, vp, ll, ll, ll, ll, ci, ci, ci, ci, ci, ci,
                                          ci, vp, vp, ll, vp]),
    "af2_template_embed": (ci, [vp, vp, vp, vp, ll, ci, ci, vp, ll, vp]),
    "af2_template_embed_workspace": (ll, [ll, ci]),
    "af2_template_embed_strict": (ci, [vp, vp, vp, vp, ll, ci, ci, vp, ll, vp]),
    "af2_template_embed_strict_workspace": (ll, [ll, ci]),
    "af2_template_angles": (ci, [C.POINTER(TemplateAngleWeights), vp, vp, ci, ci, ci, ci, ci, ci, ci, vp, ll, vp]),
    "af2_template_angles_workspace": (ll, [ci, ci, ci, ci, ci]),
    "af2_template_angles_strict": (ci, [C.POINTER(TemplateAngleWeightsStrict), vp, vp, ci, ci, ci, ci, ci, ci, ci, vp, ll, vp]),
    "af2_template_angles_strict_workspace": (ll, [ci, ci, ci, ci, ci]),
    # structure module (alphafold2.py:841-891)
    "af2_structure_linear": (ci, [vp, vp, vp, vp, ll, ci, ci, ci, vp]),
    "af2_ipa_tile_rows": (ci, [ci, ci, C.POINTER(ci)]),
    "af2_ipa_frames": (ci, [vp, vp, vp, ll, ci, vp]),
    "af2_ipa_attention": (ci, [vp, vp, vp, vp, vp, vp, vp, vp, vp, ci, ci, ci, ci, vp]),
    "af2_structure_tail": (ci, [vp, vp, vp, vp, cf, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, ll, ci, vp]),
    "af2_structure_layer_workspace": (ll, [ci, ci, ci, ci]),
    "af2_structure_layer": (ci, [C.POINTER(StructureWeights), vp, vp, vp, vp, vp, vp, vp, vp, ci, ci, ci, ci, cf, vp, ll, vp]),
    "af2_ipa_attention_rows": (ci, [vp, vp, vp, vp, vp, vp, vp, vp, vp, ci, ci, ci, ci, ci, vp]),
    "af2_structure_layer_rows_workspace": (ll, [ci, ci, ci, ci]),
    "af2_structure_layer_rows_begin": (ci, [C.POINTER(StructureWeights), vp, vp, vp, vp, vp, vp, vp, ci, ci, ci, ci, ci, vp, ll, vp]),
    "af2_structure_layer_rows_end": (ci, [C.POINTER(StructureWeights), vp, vp, vp, vp, vp, vp, vp, ci, ci, ci, cf, vp, ll, vp]),
    # peer-memory exchange of the sharded trunk
    "af2_peer_ctrl_bytes": (ci, []),
    "af2_peer_can_access": (ci, [ci, ci]),
    "af2_peer_alloc": (ci, [ll, C.POINTER(vp)]),
    "af2_peer_free": (ci, [vp]),
    "af2_peer_export": (ci, [vp, vp]),
    "af2_peer_open": (ci, [vp, C.POINTER(vp)]),
    "af2_peer_close": (ci, [vp]),
    "af2_peer_error": (ci, [vp]),
    "af2_peer_exchange": (ci, [vp, ll, ll, vp, ll, ll, ci, ll, ci, ci, ci, vp]),
    "af2_peer_exchange_chunks": (ci, [vp, ll, C.POINTER(PeerChunk), vp, ci, ci, ci, vp]),
    # distogram to coordinates (utils.py:718-833)
    "af2_center_distogram": (ci, [vp, vp, cf, vp, vp, vp, ci, ci, ci, ci, ci, ci, vp]),
    "af2_mds_workspace": (ll, [ci, ci, ci]),
    "af2_mds_iterate": (ci, [vp, vp, vp, vp, vp, vp, ci, ci, ci, C.c_double, vp, ll, vp]),
    # structure scores (utils.py:999-1247)
    "af2_metrics_workspace": (ll, [ci, ci]),
    "af2_pair_distance_scores": (ci, [ci, C.POINTER(Points), ci, C.POINTER(Points), ci, vp, ll, ll, ci, ci, cf, cf, cf, cf, vp, vp, ll,
                                      vp]),
    "af2_superpose_scores": (ci, [C.POINTER(Points), C.POINTER(Points), vp, ll, ll, ci, ci, ci, ci, C.POINTER(Points),
                                  C.POINTER(Points), vp, vp, vp, ci, C.POINTER(cf), C.POINTER(GdtSpec), ci, vp, vp, vp, ll, vp]),
    # distogram loss (train_pre.py:76-90, utils.py:45-50)
    "af2_distogram_xent_rows": (ci, [vp, vp, ci, vp, vp, ci, ci, ci, ci, ci, ll, vp, vp]),
    "af2_distogram_xent_finish": (ci, [vp, ll, vp, vp]),
    "af2_bucketed_distance": (ci, [vp, ci, vp, vp, ci, ci, ci, ll, vp, vp]),
    # angle-head labels and loss (trRosetta orientations from the backbone, DESIGN.md §4f)
    "af2_angle_xent_rows": (ci, [vp, vp, vp, vp, ci, vp, vp, ci, ci, ci, ci, ll, vp, vp]),
    "af2_angle_xent_finish": (ci, [vp, ll, vp, vp]),
    "af2_bucketed_angles": (ci, [vp, ci, vp, vp, ci, ci, ll, vp, vp, vp, vp]),
}

EXPORTED_SYMBOLS = tuple(_SIGNATURES)


def load():
    """Load the shared library (once).  Raises RuntimeError if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.isfile(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(nvcc, sm_90a). alphafold2_b200 has no CPU or PyTorch fallback.")
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def check(code: int):
    if code != 0:
        msg = load().af2_last_error().decode("utf-8", "replace")
        if code == -1:
            raise ValueError(f"af2b200: {msg}")
        raise RuntimeError(f"af2b200 (code {code}): {msg}")
