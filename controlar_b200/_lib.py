"""ctypes binding of include/controlar_b200.h.  There is NO fallback: if the CUDA library is missing or a call
fails, the product path raises."""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "lib", "libcontrolar_b200.so")

CAR_BF16, CAR_F32 = 0, 1


class CarModelDesc(C.Structure):
    _fields_ = [("dtype", C.c_int32), ("dim", C.c_int32), ("n_layer", C.c_int32), ("n_head", C.c_int32),
                ("ffn_dim", C.c_int32), ("vocab_size", C.c_int32), ("cls_token_num", C.c_int32),
                ("block_size", C.c_int32), ("caption_dim", C.c_int32), ("model_type", C.c_int32),
                ("norm_eps", C.c_float), ("rope_base", C.c_float)]


class CarWeights(C.Structure):
    _fields_ = [("tok_embeddings", C.c_void_p), ("norm", C.c_void_p), ("output", C.c_void_p),
                ("attention_norm", C.POINTER(C.c_void_p)), ("wqkv", C.POINTER(C.c_void_p)),
                ("wo", C.POINTER(C.c_void_p)), ("ffn_norm", C.POINTER(C.c_void_p)),
                ("w1", C.POINTER(C.c_void_p)), ("w3", C.POINTER(C.c_void_p)), ("w2", C.POINTER(C.c_void_p)),
                ("cap_fc1", C.c_void_p), ("cap_fc2", C.c_void_p), ("label_table", C.c_void_p),
                ("cond_fc1", C.c_void_p), ("cond_fc2", C.c_void_p),
                ("ctl_fc1", C.c_void_p * 3), ("ctl_fc2", C.c_void_p * 3)]


class CarTrainWeights(C.Structure):
    _fields_ = [("w", CarWeights), ("adapter_fc1", C.c_void_p), ("adapter_fc2", C.c_void_p), ("cap_uncond", C.c_void_p),
                ("adapter_dim", C.c_int32), ("num_classes", C.c_int32), ("cond_uncond", C.c_void_p)]


class CarTrainDropout(C.Structure):
    _fields_ = [("token_p", C.c_float), ("resid_p", C.c_float), ("ffn_p", C.c_float), ("n_layer", C.c_int32),
                ("drop_path", C.c_void_p), ("seed", C.c_void_p)]


class CarSampling(C.Structure):
    _fields_ = [("temperature", C.c_float), ("top_k", C.c_int32), ("top_p", C.c_float),
                ("sample_logits", C.c_int32), ("cfg_scale", C.c_float), ("cfg_interval", C.c_int32),
                ("seed", C.c_uint64)]


class CarRowSampling(C.Structure):
    _fields_ = [("temperature", C.c_float), ("top_k", C.c_int32), ("top_p", C.c_float), ("sample_logits", C.c_int32),
                ("seed", C.c_uint64), ("noise_row", C.c_uint32), ("control_strength", C.c_float)]


class CarDptDesc(C.Structure):
    _fields_ = [("hidden", C.c_int32), ("n_layers", C.c_int32), ("n_heads", C.c_int32), ("mlp", C.c_int32),
                ("out_indices", C.c_int32 * 4), ("neck", C.c_int32 * 4), ("fusion", C.c_int32), ("pos_grid", C.c_int32),
                ("ln_eps", C.c_float)]


class CarGemmDesc(C.Structure):
    """gemm.h's DenseP, field for field (include/controlar_b200.h)."""
    _fields_ = [("A", C.c_void_p), ("B", C.c_void_p), ("M", C.c_int32), ("N", C.c_int32), ("K", C.c_int32),
                ("lda", C.c_int32), ("ldb", C.c_int32), ("sA", C.c_int64), ("sB", C.c_int64), ("sC", C.c_int64), ("sR", C.c_int64),
                ("amode", C.c_int32), ("Hs", C.c_int32), ("Ws", C.c_int32), ("Cin", C.c_int32), ("Ho", C.c_int32), ("Wo", C.c_int32),
                ("ups", C.c_int32), ("alpha", C.c_float), ("bias", C.c_void_p), ("bias_along_m", C.c_int32), ("bias_f", C.c_void_p),
                ("resid_f", C.c_void_p), ("act", C.c_int32), ("scale", C.c_void_p), ("resid", C.c_void_p), ("ldr", C.c_int32),
                ("C", C.c_void_p), ("ldc", C.c_int32), ("out_mode", C.c_int32), ("kh", C.c_int32), ("kw", C.c_int32), ("ws", C.c_int32),
                ("osy", C.c_int32), ("osx", C.c_int32), ("oay", C.c_int32), ("oax", C.c_int32), ("oH", C.c_int32), ("oW", C.c_int32)]


class CarDinoDesc(C.Structure):
    _fields_ = [("dtype", C.c_int32), ("hidden", C.c_int32), ("heads", C.c_int32), ("layers", C.c_int32),
                ("patch", C.c_int32), ("pos_grid", C.c_int32), ("resize_mode", C.c_int32),
                ("adapter_out_dim", C.c_int32), ("eps", C.c_float)]


_DINO_ARRAYS = ["n1_w", "n1_b", "q_w", "q_b", "k_w", "k_b", "v_w", "v_b", "o_w", "o_b", "ls1", "n2_w", "n2_b",
                "fc1_w", "fc1_b", "fc2_w", "fc2_b", "ls2"]


class CarDinoWeights(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ["cls_token", "pos_emb", "patch_w", "patch_b", "ln_w", "ln_b"]] + \
               [(n, C.POINTER(C.c_void_p)) for n in _DINO_ARRAYS] + \
               [("adapter_fc1", C.c_void_p), ("adapter_fc2", C.c_void_p)]


class CarVQDesc(C.Structure):
    _fields_ = [("codebook_size", C.c_int32), ("embed_dim", C.c_int32), ("ch", C.c_int32), ("z_channels", C.c_int32),
                ("n_levels", C.c_int32), ("num_res_blocks", C.c_int32), ("ch_mult", C.c_int32 * 8)]


class CarT5Desc(C.Structure):
    _fields_ = [("dtype", C.c_int32), ("d_model", C.c_int32), ("d_kv", C.c_int32), ("n_heads", C.c_int32), ("d_ff", C.c_int32),
                ("n_layers", C.c_int32), ("vocab", C.c_int32), ("num_buckets", C.c_int32), ("max_distance", C.c_int32), ("eps", C.c_float)]


class CarT5Weights(C.Structure):
    _fields_ = [("embed", C.c_void_p), ("rel_bias", C.c_void_p), ("final_norm", C.c_void_p)] + \
               [(n, C.POINTER(C.c_void_p)) for n in ("ln1", "q", "k", "v", "o", "ln2", "wi_0", "wi_1", "wo")]


# name -> (restype, argtypes); every symbol declared in include/controlar_b200.h
PROTOTYPES = {
    "car_last_error": (C.c_char_p, []),
    "car_version": (C.c_int, []),
    "car_model_create": (C.c_int, [C.POINTER(CarModelDesc), C.POINTER(CarWeights), C.c_void_p, C.POINTER(C.c_void_p)]),
    "car_model_repack": (C.c_int, [C.c_void_p, C.POINTER(CarWeights), C.c_void_p]),
    "car_model_destroy": (C.c_int, [C.c_void_p]),
    "car_state_create": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_void_p),
                                   C.POINTER(C.c_void_p), C.c_void_p, C.POINTER(C.c_void_p)]),
    "car_state_set_emb_mask": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "car_state_set_row_sampling": (C.c_int, [C.c_void_p, C.POINTER(CarRowSampling), C.c_int32]),
    "car_state_destroy": (C.c_int, [C.c_void_p]),
    "car_state_set_step_timer": (C.c_int, [C.c_void_p, C.c_void_p]),
    "car_prefill": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p, C.c_int32, C.c_void_p]),
    "car_decode_step": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    "car_sample": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.POINTER(CarSampling), C.c_int32, C.c_int32,
                             C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "car_sample_rows": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.POINTER(CarRowSampling), C.c_int32, C.c_float, C.c_int32,
                                  C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "car_generate": (C.c_int, [C.c_void_p, C.POINTER(CarSampling), C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "car_generate_forced": (C.c_int, [C.c_void_p, C.POINTER(CarSampling), C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_void_p]),
    "car_decode_step_bytes": (C.c_int64, [C.c_void_p, C.c_int32]),
    "car_launch_count": (C.c_int64, [C.c_int32]),
    "car_op_linear": (C.c_int, [C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                C.c_int32, C.c_int32, C.c_void_p]),
    "car_op_dense_linear": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                      C.c_void_p]),
    "car_train_create": (C.c_int, [C.POINTER(CarModelDesc), C.POINTER(CarTrainWeights), C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                   C.POINTER(C.c_void_p)]),
    "car_train_forward": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "car_train_backward": (C.c_int, [C.c_void_p, C.POINTER(CarTrainWeights), C.c_void_p, C.c_void_p, C.c_void_p]),
    "car_train_destroy": (C.c_int, [C.c_void_p]),
    "car_train_set_dropout": (C.c_int, [C.c_void_p, C.POINTER(CarTrainDropout)]),
    "car_dropout_keep_mask": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_void_p,
                                        C.c_void_p]),
    "car_canny_workspace_bytes": (C.c_int64, [C.c_int32, C.c_int32]),
    "car_canny_u8": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                               C.c_void_p, C.c_void_p]),
    "car_left_pad_captions": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "car_hed_create": (C.c_int, [C.POINTER(C.c_void_p), C.c_int32, C.c_void_p, C.POINTER(C.c_void_p)]),
    "car_hed_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "car_hed_destroy": (C.c_int, [C.c_void_p]),
    "car_lineart_create": (C.c_int, [C.POINTER(C.c_void_p), C.c_int32, C.c_void_p, C.POINTER(C.c_void_p)]),
    "car_lineart_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "car_lineart_destroy": (C.c_int, [C.c_void_p]),
    "car_dpt_create": (C.c_int, [C.POINTER(CarDptDesc), C.POINTER(C.c_void_p), C.c_int32, C.c_void_p, C.POINTER(C.c_void_p)]),
    "car_dpt_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "car_dpt_destroy": (C.c_int, [C.c_void_p]),
    "car_midas_create": (C.c_int, [C.POINTER(C.c_void_p), C.c_int32, C.c_void_p, C.POINTER(C.c_void_p)]),
    "car_midas_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "car_midas_destroy": (C.c_int, [C.c_void_p]),
    "car_dino_create": (C.c_int, [C.POINTER(CarDinoDesc), C.POINTER(CarDinoWeights), C.c_void_p, C.POINTER(C.c_void_p)]),
    "car_dino_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p]),
    "car_dino_destroy": (C.c_int, [C.c_void_p]),
    "car_dino_train_create": (C.c_int, [C.POINTER(CarDinoDesc), C.POINTER(CarDinoWeights), C.c_void_p, C.POINTER(C.c_void_p)]),
    "car_dino_train_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "car_dino_train_backward": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(CarDinoWeights), C.c_void_p]),
    "car_dino_train_destroy": (C.c_int, [C.c_void_p]),
    "car_vq_create": (C.c_int, [C.POINTER(CarVQDesc), C.POINTER(C.c_void_p), C.c_int32, C.c_void_p, C.POINTER(C.c_void_p)]),
    "car_vq_decode_code": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "car_vq_decode": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "car_resize_bilinear_aa": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_int32,
                                         C.c_void_p, C.c_void_p]),
    "car_vq_encode": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "car_vq_destroy": (C.c_int, [C.c_void_p]),
    "car_t5_create": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.POINTER(C.c_void_p)]),
    "car_t5_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "car_t5_destroy": (C.c_int, [C.c_void_p]),
    "car_adamw_step": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int32, C.c_void_p]),
    "car_op_gemm_route": (C.c_int, [C.POINTER(CarGemmDesc), C.c_int32]),
    "car_op_gemm": (C.c_int, [C.POINTER(CarGemmDesc), C.c_int32, C.c_void_p]),
    "car_op_gemm_f32": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                                  C.c_void_p]),
    "car_op_gemm_f32_conv3": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                        C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "car_op_rmsnorm": (C.c_int, [C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_float,
                                 C.c_void_p]),
    "car_op_attn_decode": (C.c_int, [C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32,
                                     C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "car_op_attn_prefill": (C.c_int, [C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                      C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
}

_lib = None


def lib():
    """Load the library (once).  Raises if it has not been built — there is no CPU or eager fallback."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: build it with `python -m controlar_b200.build` "
                "(controlar_b200 has no CPU / eager-PyTorch fallback)")
        l = C.CDLL(LIB_PATH)
        for name, (res, args) in PROTOTYPES.items():
            fn = getattr(l, name)
            fn.restype = res
            fn.argtypes = args
        _lib = l
    return _lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = lib().car_last_error()
        raise RuntimeError(f"controlar_b200 {what} failed (rc={rc}): {msg.decode() if msg else '?'}")


def dtype_code(dt) -> int:
    import torch
    if dt == torch.bfloat16:
        return CAR_BF16
    if dt == torch.float32:
        return CAR_F32
    raise RuntimeError(f"controlar_b200 supports bf16 and fp32 checkpoints, not {dt}")


def cur_stream(device=None) -> int:
    """Raw handle of torch's current stream on `device` (default: the current device)."""
    import torch
    return torch.cuda.current_stream(device).cuda_stream


def on_own_device(fn):
    """Run a handle method with `self.device` current: the library launches on the current device and `cur_stream()` is that
    device's current stream, so a model on cuda:1 works without torch.cuda.set_device(1) (the reference wraps its calls in
    `with torch.device(device)`, generate.py:179-182)."""
    import functools

    @functools.wraps(fn)
    def wrapped(self, *a, **k):
        import torch
        dev = self.device
        if dev.type != "cuda":
            return fn(self, *a, **k)
        with torch.cuda.device(dev):
            return fn(self, *a, **k)
    return wrapped


def _no_handle():
    return None


class NativeHandle:
    """Owner of one library pointer, released by the entry point named `destroy` (e.g. "car_hed_destroy").  `close()` clears the
    pointer before it destroys it, so a failed re-create leaves no stale pointer and every pointer is destroyed exactly once.
    Handles are never copied: `copy.deepcopy` / pickling of the owning module (e.g. `ema = deepcopy(model)` of the train scripts,
    train_c2i_canny.py:117, after the model has been used) yields None in the copy, which rebuilds its own handle lazily on first
    use — instead of ctypes' "objects containing pointers cannot be pickled"."""

    def __init__(self, destroy: str):
        self.destroy = destroy
        self.handle = C.c_void_p()

    def close(self):
        h, self.handle = self.handle, C.c_void_p()
        if h:
            getattr(lib(), self.destroy)(h)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __deepcopy__(self, memo):
        return None

    def __reduce__(self):
        return (_no_handle, ())


def param_signature(params) -> tuple:
    """What a handle built from `params` depends on: replacing, updating in place, casting or moving a parameter changes it."""
    return tuple((p.data_ptr(), p._version, p.dtype, str(p.device)) for p in params)


class ModuleHandle(NativeHandle):
    """A library handle built from a module's parameters.  `get(params, create)` returns it, built first by `create(out)` — which
    fills the c_void_p `out` — with the parameters' device current, and built again whenever `param_signature(params)` changed."""

    def __init__(self, destroy: str):
        super().__init__(destroy)
        self.sig = None

    def get(self, params, create):
        import torch
        sig = param_signature(params)
        if not self.handle or sig != self.sig:
            if params[0].device.type != "cuda":
                raise RuntimeError("controlar_b200: the module's parameters must be on a CUDA device (there is no CPU path)")
            self.close()
            with torch.cuda.device(params[0].device):
                create(self.handle)
                torch.cuda.current_stream().synchronize()      # the library has copied / packed what it read
            self.sig = sig
        return self.handle


def _ptr(t):
    """Device pointer of a contiguous CUDA tensor (None passes through)."""
    if t is None:
        return None
    if not t.is_cuda:
        raise RuntimeError("controlar_b200: tensor is not on a CUDA device (there is no CPU fallback)")
    if not t.is_contiguous():
        raise RuntimeError("controlar_b200: tensor must be contiguous")
    return t.data_ptr()


def _ptr_array(ts):
    arr = (C.c_void_p * len(ts))()
    for i, t in enumerate(ts):
        arr[i] = _ptr(t)
    return arr


def fill_struct(struct_type, entries, layers: int = 0):
    """A `struct_type` pointing at the tensors of `entries`, and those tensors, which must stay alive while the library reads them.
    An entry is (field, index, tensor or None); a dotted field ("w.wqkv") reaches into a nested struct.  The field's ctypes type
    says what `index` is: ignored for a pointer, the slot of an inline array (`ctl_fc1[3]`), the layer of a per-layer
    POINTER(c_void_p) array.  Per-layer arrays have `layers` entries and are kept alive by the struct.  Fields, slots and layers
    that no entry names, or whose tensor is None, stay NULL."""
    s, tensors, arrays = struct_type(), [], {}
    for field, i, t in entries:
        owner = s
        *path, name = field.split(".")
        for f in path:
            owner = getattr(owner, f)
        kind = dict(owner._fields_)[name]
        p = _ptr(t)
        if t is not None:
            tensors.append(t)
        if kind is C.c_void_p:
            setattr(owner, name, p)
        elif issubclass(kind, C.Array):
            getattr(owner, name)[i] = p
        else:
            if field not in arrays:
                arrays[field] = (C.c_void_p * layers)()
                setattr(owner, name, C.cast(arrays[field], C.POINTER(C.c_void_p)))
            arrays[field][i] = p
    return s, tensors
