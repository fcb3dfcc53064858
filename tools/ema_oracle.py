"""NumPy restatement of the weight EMA (models/ema.py ModelEma, csrc/optim.cu multi_ema_kernel).
tests/test_model_ema.py compares the kernel and the graphed training step against it bit for bit, and pins it to a
literal transcription of TF's assign_moving_average with the num_updates ramp.

  decay_at   d = ramp ? min(decay, (1 + k) / (10 + k)) : decay, in fp64, for update number k >= 1
  weight     w = (float32)(1 - d), rounded once
  update     e - w * (e - s) in float32, each operation rounded on its own
  apply      update over a dict or list of arrays, for update number k
"""
import numpy as np


def decay_at(decay, k, ramp=True):
    """TF's ExponentialMovingAverage(decay, num_updates=k) with Python floats (fp64)"""
    decay = float(decay)
    return min(decay, (1.0 + k) / (10.0 + k)) if ramp else decay


def weight(decay, k, ramp=True):
    return np.float32(1.0 - decay_at(decay, k, ramp))


def update(e, s, w):
    """e, s float32 arrays (s broadcast to e's shape), w float32 -> the averaged array, float32"""
    e = np.asarray(e, dtype=np.float32)
    s = np.asarray(s, dtype=np.float32)
    diff = (e - s).astype(np.float32)
    return (e - (np.float32(w) * diff).astype(np.float32)).astype(np.float32)


def apply(ema, src, k, decay, ramp=True):
    """ema, src: dicts (or lists) of float32 arrays -> the same structure after update number k"""
    w = weight(decay, k, ramp)
    if isinstance(ema, dict):
        return {n: update(ema[n], src[n], w) for n in ema}
    return [update(e, s, w) for e, s in zip(ema, src)]
