"""Float64 NumPy reference of the six Keras learning-rate schedules (tf.keras 2.13+ / Keras 3), written from their
definitions: `step` is the number of updates already applied.  Independent of tf_yarn_b200."""
import math

import numpy as np


def exponential(step, initial, decay_steps, decay_rate, staircase=False):
    p = np.float64(step) / decay_steps
    if staircase:
        p = np.floor(p)
    return initial * np.power(np.float64(decay_rate), p)


def piecewise(step, boundaries, values):
    # values[0] while step <= boundaries[0], values[i] while boundaries[i-1] < step <= boundaries[i], values[-1] after
    for b, v in zip(boundaries, values):
        if step <= b:
            return np.float32(v)
    return np.float32(values[-1])


def polynomial(step, initial, decay_steps, end=1e-4, power=1.0, cycle=False):
    step = np.float64(step)
    if cycle:
        d = decay_steps * max(1.0, math.ceil(step / decay_steps))
    else:
        d, step = decay_steps, min(step, decay_steps)
    return (initial - end) * (1.0 - step / d) ** power + end


def inverse_time(step, initial, decay_steps, decay_rate, staircase=False):
    p = np.float64(step) / decay_steps
    if staircase:
        p = np.floor(p)
    return initial / (1.0 + decay_rate * p)


def _cos_decay(t, decay_steps, alpha, from_lr):
    return from_lr * ((1.0 - alpha) * 0.5 * (1.0 + np.cos(np.pi * t / decay_steps)) + alpha)


def cosine(step, initial, decay_steps, alpha=0.0, warmup_target=None, warmup_steps=0):
    step = np.float64(step)
    if warmup_target is None:
        return _cos_decay(min(step, decay_steps), decay_steps, alpha, initial)
    t = min(step, decay_steps + warmup_steps)
    if t < warmup_steps:
        return initial + (warmup_target - initial) * t / warmup_steps
    return _cos_decay(t - warmup_steps, decay_steps, alpha, warmup_target)


def cosine_restarts(step, initial, first_decay_steps, t_mul=2.0, m_mul=1.0, alpha=0.0):
    """Period i lasts first_decay_steps * t_mul**i steps; walk the periods in steps."""
    start, length, i = 0.0, float(first_decay_steps), 0
    if t_mul == 1.0:
        i = math.floor(step / first_decay_steps)
        start = i * first_decay_steps
    else:
        while step >= start + length:
            start += length
            length *= t_mul
            i += 1
    frac = (step - start) / length
    return initial * ((1.0 - alpha) * 0.5 * m_mul ** i * (1.0 + np.cos(np.pi * frac)) + alpha)
