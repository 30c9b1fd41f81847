"""Channel statistics for the standardised observation (the reference's normalize.py and transform_observation(normalize=False)).

normalize.py (:20-66) takes np.mean / np.std (population) of every pixel of 100 reset observations per channel and pickles
[mean_r, mean_g, mean_b, mean_d, std_r, std_g, std_b, std_d] to `mean_and_std`: the RGB entries are np.float64 (numpy reduces uint8
input in float64), the depth entries np.float32 (float32 input is reduced in float32).  Grasp_Agent.get_mean_std (:370-379) reads
that file back as values[0:4], values[4:8].

* `channel_statistics(rgb, depth)` computes the eight values of a batch of device observations with gq_obs_channel_stats: the RGB
  means bit for bit numpy's, the RGB stds from exact integer sums (closer to the exact value than numpy's pairwise sum of squared
  deviations, which differs in the last bits), the depth values in fp64 rounded once to f32 (numpy's float32 pairwise sums differ
  from them in the last float32 bits).  DESIGN.md section 2, decision 11.
* `save_mean_and_std` / `load_mean_and_std` write and read the reference's pickle, so a file of either side works on the other.
* `check_mean_and_std` is what every consumer runs on the values before it uses them.
"""
import math
import pickle

import numpy as np

_NUMPY_SCALAR = {("numpy.core.multiarray", "scalar"), ("numpy._core.multiarray", "scalar"), ("numpy", "dtype")}


class _ScalarUnpickler(pickle.Unpickler):
    """reads a list of numpy scalars and nothing else: a `mean_and_std` file cannot make the loader run other code"""

    def find_class(self, module, name):
        if (module, name) in _NUMPY_SCALAR:
            return np.dtype if name == "dtype" else _numpy_scalar()
        raise pickle.UnpicklingError(f"a mean_and_std file holds numpy scalars only, not {module}.{name}")


def _numpy_scalar():
    try:
        from numpy._core.multiarray import scalar
    except ImportError:  # numpy < 2
        from numpy.core.multiarray import scalar
    return scalar


def _typed(values):
    """-> the eight values as the reference's types ([f64 x3, f32, f64 x3, f32]); ValueError unless there are eight finite numbers"""
    try:
        v = [float(x) for x in values]
    except (TypeError, ValueError):
        raise ValueError(f"mean_and_std must be 8 numbers (mean r, g, b, depth, std r, g, b, depth), not {values!r}") from None
    if len(v) != 8 or not all(math.isfinite(x) for x in v):
        raise ValueError(f"mean_and_std must be 8 finite numbers (mean r, g, b, depth, std r, g, b, depth), got {len(v)}: {v}")
    return [np.float64(v[0]), np.float64(v[1]), np.float64(v[2]), np.float32(v[3]), np.float64(v[4]), np.float64(v[5]), np.float64(v[6]), np.float32(v[7])]


def check_mean_and_std(values):
    """-> the eight values with the reference's types; ValueError unless they are eight finite numbers whose four standard deviations
    are > 0 in float32, the precision the transform uses (torchvision's Normalize refuses a zero std)"""
    v = _typed(values)
    if any(not np.float32(s) > 0 for s in v[4:]):
        raise ValueError(f"every standard deviation of mean_and_std must be > 0, got {[float(s) for s in v[4:]]}")
    return v


def as_float32(values):
    """the eight values as the transform uses them: float32, as torchvision's Normalize converts mean and std to the tensor's dtype"""
    return np.asarray([np.float32(x) for x in check_mean_and_std(values)], dtype=np.float32)


def save_mean_and_std(path, values):
    """writes the reference's `mean_and_std` pickle (normalize.py:60-64): a list of 8 numpy scalars, f64 for RGB, f32 for depth"""
    vals = check_mean_and_std(values)
    with open(path, "wb") as f:
        pickle.dump(vals, f)
    return vals


def load_mean_and_std(path):
    """reads a `mean_and_std` pickle (the reference's own or save_mean_and_std's) -> the list of 8 values with the reference's types"""
    with open(path, "rb") as f:
        try:
            raw = _ScalarUnpickler(f).load()
        except (pickle.UnpicklingError, EOFError) as e:
            raise ValueError(f"{path} is not a mean_and_std file: {e}") from None
    if not isinstance(raw, list):
        raise ValueError(f"{path}: a mean_and_std file holds a list of 8 values, not {type(raw).__name__}")
    return check_mean_and_std(raw)


def channel_statistics(rgb, depth):
    """normalize.py's eight statistics of B observations on the device (gq_obs_channel_stats): rgb u8 [B,H,W,3], depth f32 [B,H,W]
    metres, the same CUDA device -> [mean_r, mean_g, mean_b, mean_d, std_r, std_g, std_b, std_d] with the reference's types"""
    import ctypes as C

    import torch

    from .qnet import load_qnet_library

    if not (rgb.is_cuda and depth.is_cuda) or rgb.device != depth.device:
        raise ValueError("channel_statistics needs rgb and depth on one CUDA device (there is no CPU fallback)")
    if rgb.dtype != torch.uint8 or depth.dtype != torch.float32 or rgb.dim() != 4 or rgb.shape[3] != 3 or tuple(rgb.shape[:3]) != tuple(depth.shape):
        raise ValueError(f"channel_statistics takes rgb u8 [B,H,W,3] and depth f32 [B,H,W], got {rgb.dtype} {tuple(rgb.shape)}, {depth.dtype} {tuple(depth.shape)}")
    L = load_qnet_library()
    rgb, depth = rgb.contiguous(), depth.contiguous()
    B, HW = depth.shape[0], depth.shape[1] * depth.shape[2]
    scratch = torch.empty(L.gq_obs_channel_stats_scratch_bytes(B * HW), dtype=torch.uint8, device=depth.device)
    out = torch.empty(8, dtype=torch.float64, device=depth.device)
    stream = torch.cuda.current_stream(depth.device).cuda_stream
    r = L.gq_obs_channel_stats(C.c_void_p(rgb.data_ptr()), C.c_void_p(depth.data_ptr()), B, HW, C.c_void_p(scratch.data_ptr()), C.c_void_p(out.data_ptr()),
                               C.c_void_p(stream))
    if r != 0:
        raise RuntimeError(f"gq_obs_channel_stats failed ({r}): {L.gq_last_error().decode()}")
    return _typed(out.cpu().tolist())
