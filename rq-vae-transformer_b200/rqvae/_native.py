"""ctypes binding of the C ABI in include/rqb200.h (csrc/librqb200.so).  Fails loudly when the library is absent."""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("RQB200_LIB", os.path.join(os.path.dirname(_HERE), "csrc", "librqb200.so"))

OK, EINVAL, ECUDA, ENODEV, EWORKSPACE, ESTATE = 0, -1, -2, -3, -4, -5
F32, BF16, F16, E4M3 = 0, 1, 2, 3
MODE_EXACT, MODE_FAST = 0, 1
AR_NO_GRAPH, AR_NO_PDL, AR_TRACE, AR_SEQUENTIAL_PREFILL = 1, 2, 4, 32
# rqb200_ar_config.embed_variant bits (0 = the shipped family)
EMB_TOK_INPUT, EMB_TOK_HEAD, EMB_NO_CUMSUM, EMB_TUPLE, EMB_CLS_PER_DEPTH = 1, 2, 4, 8, 16
_DT = {torch.float32: F32, torch.bfloat16: BF16, torch.float16: F16}

c_f32p, c_i64p, c_vp = C.c_void_p, C.c_void_p, C.c_void_p


class BlockWeights(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("wqkv", "wproj", "w1", "w2", "bqkv", "bproj", "b1", "b2",
                                          "ln1_w", "ln1_b", "ln2_w", "ln2_b", "sqkv", "sproj", "s1", "s2")]


class ArConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("embed_dim", "n_head", "n_body", "n_head_layers", "vocab", "H", "W", "D",
                                         "vocab_cond", "cond_len", "code_dim", "codebook_size", "mode", "weight_dtype",
                                         "flags", "split_qkv", "split_proj", "split_fc1", "split_fc2",
                                         "codebook_per_depth", "embed_variant")]


class ArWeights(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("pos_emb_cond", "pos_emb_hw", "pos_emb_d", "cond_emb", "w_in", "w_head", "w_cls",
                                          "b_in", "b_head", "b_cls", "cls_ln_w", "cls_ln_b", "codebook")] + \
               [("body", C.POINTER(BlockWeights)), ("head", C.POINTER(BlockWeights))] + \
               [(n, C.c_void_p) for n in ("w_ccls", "b_ccls", "ccls_ln_w", "ccls_ln_b", "tok_emb", "s_in", "s_head", "s_cls", "s_ccls")]


class VaeConfig(C.Structure):
    _fields_ = [("ch", C.c_int32), ("n_levels", C.c_int32), ("ch_mult", C.c_int32 * 8), ("num_res_blocks", C.c_int32),
                ("n_attn_res", C.c_int32), ("attn_resolutions", C.c_int32 * 8), ("resolution", C.c_int32),
                ("z_channels", C.c_int32), ("embed_dim", C.c_int32), ("in_channels", C.c_int32), ("out_ch", C.c_int32),
                ("codebook_size", C.c_int32), ("depth", C.c_int32), ("mode", C.c_int32)]


_lib = None


class NativeError(RuntimeError):
    pass


def lib():
    """Loads librqb200.so once.  No fallback: a missing library is a hard error."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise NativeError("rqb200: native library not found at %s -- build it with "
                          "rq-vae-transformer_b200/csrc/build.sh (or __graft_entry__.build()); there is no CPU fallback"
                          % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    L.rqb200_last_error.restype = C.c_char_p
    L.rqb200_version.restype = C.c_int
    L.rqb200_device_count.restype = C.c_int
    L.rqb200_rq_quantize.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_void_p]
    L.rqb200_rq_soft_codes.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_float, C.c_void_p, C.c_void_p,
                                       C.c_void_p]
    L.rqb200_rq_embed_sum.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    L.rqb200_rq_embed_depth.argtypes = L.rqb200_rq_embed_sum.argtypes
    # per-depth codebooks: host arrays of D device pointers and D sizes
    L.rqb200_rq_quantize_depthwise.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int32), C.c_int64, C.c_int, C.c_int,
                                               C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.rqb200_dbg_rq_quantize_depthwise.argtypes = [C.c_int] + L.rqb200_rq_quantize_depthwise.argtypes
    L.rqb200_rq_embed_sum_depthwise.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int32), C.c_int64, C.c_int, C.c_int,
                                                C.c_void_p, C.c_void_p]
    L.rqb200_rq_embed_depth_depthwise.argtypes = L.rqb200_rq_embed_sum_depthwise.argtypes
    L.rqb200_sample_logits.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_int, C.c_float, C.c_void_p,
                                       C.c_void_p]
    L.rqb200_dbg_rows_gemm.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int64,
                                       C.c_int, C.c_int, C.c_void_p]
    L.rqb200_dbg_rq_quantize.argtypes = [C.c_int] + L.rqb200_rq_quantize.argtypes
    L.rqb200_dbg_sample_logits.argtypes = [C.c_int] + L.rqb200_sample_logits.argtypes
    L.rqb200_ar_create.restype = C.c_void_p
    L.rqb200_ar_create.argtypes = [C.POINTER(ArConfig), C.POINTER(ArWeights)]
    L.rqb200_ar_destroy.argtypes = [C.c_void_p]
    L.rqb200_ar_destroy.restype = None
    L.rqb200_ar_workspace_bytes.restype = C.c_size_t
    L.rqb200_ar_workspace_bytes.argtypes = [C.c_void_p, C.c_int]
    # the arguments up to cfg_scale (ABI 113).  ABI 117 appended canvas_h and canvas_w (C int): every caller passes them after
    # these as C.c_int values, which ctypes forwards as declared-int arguments of the same call.
    L.rqb200_ar_sample_span.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float,
                                        C.POINTER(C.c_int32), C.POINTER(C.c_float), C.c_void_p, C.c_int64, C.c_void_p,
                                        C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p,
                                        C.c_void_p, C.c_void_p, C.c_int, C.c_float]
    L.rqb200_ar_step.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                 C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    L.rqb200_ar_forward_workspace_bytes.restype = C.c_size_t
    L.rqb200_ar_forward_workspace_bytes.argtypes = [C.c_void_p, C.c_int]
    L.rqb200_ar_forward.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                    C.c_void_p]
    L.rqb200_ar_log_prob_workspace_bytes.restype = C.c_size_t
    L.rqb200_ar_log_prob_workspace_bytes.argtypes = [C.c_void_p, C.c_int]
    L.rqb200_ar_log_prob.argtypes = L.rqb200_ar_forward.argtypes
    L.rqb200_dbg_log_prob_rows.argtypes = [C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]
    L.rqb200_ar_trace.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_char_p, C.c_int]
    L.rqb200_ar_last_launches.restype = C.c_int64
    L.rqb200_ar_last_launches.argtypes = [C.c_void_p]
    L.rqb200_vae_create.restype = C.c_void_p
    L.rqb200_vae_create.argtypes = [C.POINTER(VaeConfig)]
    L.rqb200_vae_destroy.argtypes = [C.c_void_p]
    L.rqb200_vae_destroy.restype = None
    L.rqb200_vae_set_tensor.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int, C.c_int64]
    L.rqb200_vae_finalize.argtypes = [C.c_void_p]
    L.rqb200_vae_workspace_bytes.restype = C.c_size_t
    L.rqb200_vae_workspace_bytes.argtypes = [C.c_void_p, C.c_int]
    for fn in (L.rqb200_vae_decode, L.rqb200_vae_decode_code, L.rqb200_vae_encode):
        fn.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    L.rqb200_vae_workspace_bytes_hw.restype = C.c_size_t
    L.rqb200_vae_workspace_bytes_hw.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int]
    for fn in (L.rqb200_vae_decode_hw, L.rqb200_vae_encode_hw):
        fn.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    L.rqb200_vae_last_launches.restype = C.c_int64
    L.rqb200_vae_last_launches.argtypes = [C.c_void_p]
    L.rqb200_dbg_gemm_tc.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p,
                                     C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
    L.rqb200_dbg_gemm_tc_fp8.argtypes = [C.c_void_p] * 6 + [C.c_int, C.c_int, C.c_void_p] + [C.c_int] * 4 + [C.c_void_p]
    L.rqb200_dbg_gemm_tc_epi.argtypes = [C.c_void_p] * 3 + [C.c_int, C.c_void_p, C.c_float, C.c_void_p, C.c_int64, C.c_int, C.c_void_p,
                                         C.c_int64, C.c_void_p, C.c_void_p] + [C.c_int] * 5 + [C.c_void_p]
    L.rqb200_dbg_conv_tc.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                     C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
    L.rqb200_dbg_conv_tc_gn.argtypes = [C.c_void_p] * 8 + [C.c_int] * 7 + [C.c_void_p]
    L.rqb200_dbg_attn_step.argtypes = [C.c_int, C.c_void_p, C.c_int] + [C.c_void_p] * 4 + [C.c_int] * 3 + [C.c_void_p] + [C.c_int] * 2 + \
                                      [C.c_void_p]
    L.rqb200_dbg_prefill_attn.argtypes = [C.c_void_p] * 4 + [C.c_int] * 5 + [C.c_void_p]
    L.rqb200_dbg_append_attn.argtypes = [C.c_void_p] * 4 + [C.c_int] * 6 + [C.c_void_p]
    L.rqb200_dbg_ln.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int] + [C.c_void_p] * 6 + [C.c_int64, C.c_int, C.c_int, C.c_void_p]
    L.rqb200_dbg_act_reduce.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p] + [C.c_int] * 3 + [C.c_void_p]
    L.rqb200_dbg_vae_conv.argtypes = [C.c_void_p, C.c_void_p, C.c_int] + [C.c_void_p] * 3 + [C.c_int] * 10 + [C.c_void_p]
    L.rqb200_dbg_groupnorm.argtypes = [C.c_int] + [C.c_void_p] * 7 + [C.c_int64] + [C.c_int] * 4 + [C.c_void_p]
    L.rqb200_dbg_cast_f16.argtypes = [C.c_void_p] * 3 + [C.c_int] * 5 + [C.c_void_p]
    L.rqb200_dbg_vae_attn.argtypes = [C.c_void_p] * 2 + [C.c_int] * 3 + [C.c_void_p]
    L.rqb200_dbg_vae_attn_tc.argtypes = [C.c_void_p] * 2 + [C.c_int] * 3 + [C.c_void_p]
    _lib = L
    return L


EXPORTS = ["rqb200_last_error", "rqb200_version", "rqb200_device_count", "rqb200_rq_quantize", "rqb200_rq_embed_sum",
           "rqb200_rq_embed_depth", "rqb200_rq_soft_codes", "rqb200_sample_logits", "rqb200_ar_create", "rqb200_ar_destroy",
           "rqb200_ar_workspace_bytes", "rqb200_ar_sample_span", "rqb200_ar_step", "rqb200_ar_forward",
           "rqb200_ar_forward_workspace_bytes", "rqb200_ar_trace", "rqb200_ar_last_launches", "rqb200_vae_create",
           "rqb200_vae_destroy", "rqb200_vae_set_tensor", "rqb200_vae_finalize", "rqb200_vae_workspace_bytes",
           "rqb200_vae_decode", "rqb200_vae_decode_code", "rqb200_vae_encode", "rqb200_vae_last_launches",
           "rqb200_dbg_gemm_tc", "rqb200_dbg_gemm_tc_fp8", "rqb200_dbg_gemm_tc_epi", "rqb200_dbg_conv_tc", "rqb200_dbg_conv_tc_gn", "rqb200_dbg_rq_quantize", "rqb200_dbg_sample_logits",
           "rqb200_dbg_rows_gemm", "rqb200_rq_quantize_depthwise", "rqb200_rq_embed_sum_depthwise",
           "rqb200_rq_embed_depth_depthwise", "rqb200_dbg_rq_quantize_depthwise", "rqb200_ar_log_prob",
           "rqb200_ar_log_prob_workspace_bytes", "rqb200_dbg_log_prob_rows", "rqb200_dbg_attn_step", "rqb200_dbg_prefill_attn", "rqb200_dbg_append_attn",
           "rqb200_dbg_ln", "rqb200_dbg_act_reduce", "rqb200_dbg_vae_conv", "rqb200_dbg_groupnorm", "rqb200_dbg_cast_f16",
           "rqb200_dbg_vae_attn", "rqb200_vae_workspace_bytes_hw", "rqb200_vae_encode_hw", "rqb200_vae_decode_hw",
           "rqb200_dbg_vae_attn_tc", "rqb200_inception_create", "rqb200_inception_destroy", "rqb200_inception_set_tensor",
           "rqb200_inception_params_bytes", "rqb200_inception_finalize", "rqb200_inception_workspace_bytes", "rqb200_inception_forward",
           "rqb200_inception_last_launches", "rqb200_dbg_inception_conv", "rqb200_dbg_inception_conv_tc", "rqb200_dbg_inception_input", "rqb200_dbg_inception_pool",
           "rqb200_dbg_inception_gap", "rqb200_clip_create", "rqb200_clip_destroy", "rqb200_clip_set_tensor", "rqb200_clip_params_bytes",
           "rqb200_clip_finalize", "rqb200_clip_workspace_bytes", "rqb200_clip_text_workspace_bytes", "rqb200_clip_encode_image",
           "rqb200_clip_encode_text", "rqb200_clip_cosine", "rqb200_clip_last_launches", "rqb200_clip_resize_plan",
           "rqb200_dbg_clip_preprocess", "rqb200_dbg_clip_attn", "rqb200_dbg_clip_attn_flash", "rqb200_lpips_create",
           "rqb200_lpips_destroy", "rqb200_lpips_set_tensor", "rqb200_lpips_params_bytes", "rqb200_lpips_finalize",
           "rqb200_lpips_workspace_bytes", "rqb200_lpips_forward", "rqb200_lpips_last_launches", "rqb200_dbg_lpips_input",
           "rqb200_dbg_lpips_pool", "rqb200_dbg_lpips_head", "rqb200_dbg_lpips_mean"]


def check(rc, what=""):
    if rc != 0:
        raise NativeError("rqb200 %s failed (%d): %s" % (what, rc, lib().rqb200_last_error().decode()))


def require_cuda(*tensors):
    """the product path is CUDA-only: refuse CPU tensors instead of silently computing elsewhere"""
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise NativeError("rqb200: tensor on %s -- this engine has no CPU path; move the model and inputs to a "
                              "CUDA device" % t.device)


def stream_ptr(device=None):
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def dtype_code(t):
    return _DT[t.dtype]


def default_precision():
    """'exact' (fp32 FFMA, bit-exact-indices gate) or 'fast' (fp16/bf16 wgmma).  RQB200_PRECISION overrides."""
    return os.environ.get("RQB200_PRECISION", "auto")


def fast_dtype():
    """16-bit activation format of the fast AR tier: fp16 (the reference's autocast class) unless RQB200_FAST_DTYPE=bf16
    (RQB200_FAST_DTYPE=fp8 keeps fp16 activations)"""
    return torch.bfloat16 if os.environ.get("RQB200_FAST_DTYPE", "fp16").lower() in ("bf16", "bfloat16") else torch.float16


def fast_weight_format():
    """weight format of the fast AR tier, read from RQB200_FAST_DTYPE (case-insensitive): 'fp8' (E4M3 values with one fp32 scale
    per output row, fp16 activations), 'bf16', or 'fp16' -- the default, also for any value it does not know"""
    v = os.environ.get("RQB200_FAST_DTYPE", "fp16").lower()
    return "fp8" if v == "fp8" else ("bf16" if v in ("bf16", "bfloat16") else "fp16")


FP8_MAX = 448.0                  # largest finite float8_e4m3fn


def quantize_fp8_rows(w):
    """FP8 (E4M3) weight format: one fp32 scale per output row, s = amax|w[n]| / 448 (s = 1 for an all-zero row), q = w / s
    clamped to +-448 and rounded to float8_e4m3fn.  Returns (q [N,K] float8_e4m3fn, s [N] f32) on w's device; q * s is the weight
    the fp8 kernels compute with.  Every step is correctly rounded, so the CPU and the GPU give the same bits (both divisions take
    a tensor divisor: CUDA torch divides by a Python scalar as a multiplication by its reciprocal)."""
    w = w.detach().float()
    amax = w.abs().amax(dim=1)
    s = amax / torch.full_like(amax, FP8_MAX)
    s = torch.where(s > 0, s, torch.ones_like(s))
    q = (w / s[:, None]).clamp(-FP8_MAX, FP8_MAX).to(torch.float8_e4m3fn)
    return q, s


_FP8_TILE = None


def fp8_tile_order():
    """[8192] int64: element (row * 64 + k) of a 128 x 64 weight tile stored at each byte of its packed form.  Packed byte
    ((wg * 2 + h) * 128 + t) * 16 + b belongs to consumer thread t of warpgroup wg, k16 step kk = 2 h + b / 8, element e = b % 8
    of the wgmma m64k16 A fragment: row 64 wg + 16 (t / 32) + (t % 32) / 4 + 8 ((e / 2) % 2), k 16 kk + 2 (t % 4) + 8 (e / 4) + e % 2."""
    global _FP8_TILE
    if _FP8_TILE is None:
        p = torch.arange(8192)
        wg, h, t, b = p // 4096, (p // 2048) % 2, (p // 16) % 128, p % 16
        kk, e, lane = 2 * h + b // 8, b % 8, t % 32
        row = 64 * wg + 16 * (t // 32) + lane // 4 + 8 * ((e // 2) % 2)
        col = 16 * kk + 2 * (lane % 4) + 8 * (e // 4) + e % 2
        _FP8_TILE = row * 64 + col
    return _FP8_TILE


def pack_fp8_tiles(q):
    """q [N,K] float8_e4m3fn (N % 128 == 0, K % 64 == 0) -> the packed uint8 weight stream of the fp8 GEMM: tile (T, kb) of rows
    [128 T, 128 T + 128) x k [64 kb, 64 kb + 64) is 8 KB at byte (T * K / 64 + kb) * 8192, in fp8_tile_order()."""
    N_out, K = q.shape
    if N_out % 128 or K % 64:
        raise ValueError("pack_fp8_tiles: need N %% 128 == 0 and K %% 64 == 0, got [%d, %d]" % (N_out, K))
    t = q.view(torch.uint8).reshape(N_out // 128, 128, K // 64, 64).permute(0, 2, 1, 3).reshape(-1, 8192)
    return t[:, fp8_tile_order().to(q.device)].reshape(-1).contiguous()


def unpack_fp8_tiles(packed, N_out, K):
    """inverse of pack_fp8_tiles: -> q [N_out,K] float8_e4m3fn"""
    t = torch.empty(N_out // 128 * (K // 64), 8192, dtype=torch.uint8, device=packed.device)
    t[:, fp8_tile_order().to(packed.device)] = packed.reshape(-1, 8192)
    return t.reshape(N_out // 128, K // 64, 128, 64).permute(0, 2, 1, 3).reshape(N_out, K).view(torch.float8_e4m3fn)


def pack_fp8_weight(w):
    """the AR engine's E4M3 form of one streamed weight, on w's device (CPU or GPU: the same bits).  w [N,K] (nn.Linear layout):
    -> (packed uint8 [N*K] in pack_fp8_tiles' order, s [N] f32).  w [D,N,K] (one [N,K] weight per depth, e.g. the per-depth
    classifiers of a BatchLinear transposed): each depth quantised by its own rows and packed on its own, the D streams concatenated
    (depth d's at byte d*N*K) -> (packed [D*N*K], s [D,N])."""
    if w.dim() == 2:
        q, s = quantize_fp8_rows(w)
        return pack_fp8_tiles(q), s
    packed, scales = zip(*(pack_fp8_weight(w[d]) for d in range(w.shape[0])))
    return torch.cat(packed), torch.stack(scales)


def ar_engine_options():
    """rqb200_ar_config.flags of the fast AR tier, read ONCE per engine from the environment (diagnostics)"""
    env = os.environ.get
    flags = 0
    flags |= AR_NO_GRAPH if env("RQB200_NO_GRAPH", "0") == "1" else 0
    flags |= AR_NO_PDL if env("RQB200_NO_PDL", "0") == "1" else 0
    flags |= AR_TRACE if env("RQB200_TRACE", "0") == "1" else 0
    flags |= AR_SEQUENTIAL_PREFILL if env("RQB200_SEQ_PREFILL", "0") == "1" else 0
    return flags


def param_fingerprint(module):
    """identity + in-place-write counter of every parameter / buffer.  The native engines cache packed weight copies; they are
    rebuilt when this changes (nested load_state_dict through a wrapper, EMA updates, optimizer steps, .data swaps)."""
    return hash(tuple((t.data_ptr(), t._version) for t in list(module.parameters()) + list(module.buffers())))


class EngineCache:
    """Mixin for an nn.Module whose forward runs in native engines built from its parameters.  The engines live in ``_eng`` (key ->
    {"handle", ...}) and are destroyed through ``_DESTROY`` (the C function's name) when the module moves (``_apply``), loads a
    state_dict, is collected, or its parameters change in a way its own hooks do not see (``_cached_engine``'s fingerprint)."""
    _DESTROY = None

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.precision = None            # None -> default_precision() ('auto' == exact unless the module says otherwise)
        self._eng = {}
        self._eng_fp = None              # the fingerprint the cached engines were built from
        self.last_launches = 0

    def _invalidate_native(self):
        for e in self._eng.values():
            getattr(lib(), self._DESTROY)(e["handle"])
        self._eng = {}

    def _apply(self, fn, *a, **k):
        self._invalidate_native()
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, *a, **k):
        self._invalidate_native()
        return super().load_state_dict(*a, **k)

    def __del__(self):
        try:
            self._invalidate_native()
        except Exception:
            pass

    def _mode(self):
        p = self.precision or default_precision()
        return MODE_FAST if p == "fast" else MODE_EXACT

    def _cached_engine(self, key, fingerprint, build):
        """the engine under key, made by build() when absent; every engine is dropped first when fingerprint differs from the one
        they were built from (weights changed behind the module's own hooks: a wrapper's load, an in-place write)"""
        if fingerprint != self._eng_fp:
            self._invalidate_native()
            self._eng_fp = fingerprint
        if key not in self._eng:
            self._eng[key] = build()
        return self._eng[key]


def bind_plan_engine(L, prefix, cfg_type):
    """ctypes signatures of the lifecycle every layer-plan engine rqb200_<prefix>_* shares: create (from a cfg_type), destroy,
    set_tensor, params_bytes, finalize and last_launches"""
    fn = lambda name: getattr(L, "rqb200_%s_%s" % (prefix, name))
    fn("create").restype = C.c_void_p
    fn("create").argtypes = [C.POINTER(cfg_type)]
    fn("destroy").argtypes = [C.c_void_p]
    fn("destroy").restype = None
    fn("set_tensor").argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int, C.c_int64]
    fn("params_bytes").restype = C.c_size_t
    fn("params_bytes").argtypes = [C.c_void_p]
    fn("finalize").argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    fn("last_launches").restype = C.c_int64
    fn("last_launches").argtypes = [C.c_void_p]


def plan_engine(L, prefix, cfg, tensors, device):
    """a layer-plan engine rqb200_<prefix>_* (L bound by bind_plan_engine) on device: created from cfg, every tensor of {key: tensor}
    registered as a contiguous fp32 copy, its parameter buffer allocated and finalized -> {"handle", "keep", "params", "ws"}"""
    fn = lambda name: getattr(L, "rqb200_%s_%s" % (prefix, name))
    handle = fn("create")(C.byref(cfg))
    if not handle:
        raise NativeError("rqb200_%s_create: %s" % (prefix, L.rqb200_last_error().decode()))
    eng = {"handle": handle, "keep": {}, "ws": None}
    try:
        for k, v in tensors.items():
            require_cuda(v)
            t = v.detach().float().contiguous()
            eng["keep"][k] = t
            check(fn("set_tensor")(handle, k.encode(), ptr(t), dtype_code(t), t.numel()), prefix + "_set_tensor")
        eng["params"] = params = torch.empty(fn("params_bytes")(handle), dtype=torch.uint8, device=device)
        with torch.cuda.device(device):
            check(fn("finalize")(handle, ptr(params), params.numel(), stream_ptr(device)), prefix + "_finalize")
    except BaseException:
        fn("destroy")(handle)
        raise
    return eng


def workspace(eng, need, device, refused=None):
    """eng["ws"] grown to at least `need` bytes on device; a growing buffer is released before the larger one is allocated.  need == 0
    is the engine refusing the call's arguments: NativeError(refused), unless refused is None and the engine's own call reports it."""
    if need == 0 and refused is not None:
        raise NativeError(refused)
    if eng["ws"] is None or eng["ws"].numel() < need:
        eng["ws"] = None
        eng["ws"] = torch.empty(need, dtype=torch.uint8, device=device)
    return eng["ws"]


launch_count = {"total": 0}      # kernels launched by our library through this binding (bench.py's gpu_launches)
