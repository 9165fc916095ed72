"""Observation corruptors for BatchedMujocoEnv.modify_observable (the reference's utils/observables.py factories).

The reference's factories return Python callables that numpy runs once per sample.  Here the noise is drawn on the device, inside
the substep loop, so the factories return SPEC objects that describe the corruptor; modify_observable uploads them as tables
(b2s_obs_modifiers, include/b2s.h).  A spec is applied to a sample as
    Gaussian: clip(v + (mean + std * z), low, high)          Uniform: clip(v + (min_noise + (max_noise - min_noise) * u), low, high)
with z ~ N(0, 1) and u ~ U[0, 1) drawn per observation row and sample.

The factories keep the reference's argument names.  Their defaults are recalled from the reference, not checked against a
checkout of it (as DEFAULT_DYNAMICS_ARGS in wrappers.py); the reference spells the factories `..._corrupter`, which this module
also provides under that spelling.
"""
import math
from dataclasses import dataclass

from .engine import CORRUPT_GAUSSIAN, CORRUPT_UNIFORM


def _check_bounds(low, high):
    if math.isnan(low) or math.isnan(high) or low > high:
        raise ValueError("corruptor clip range: low ({}) must not exceed high ({})".format(low, high))


@dataclass(frozen=True)
class GaussianNoiseCorruptor:
    """adds mean + std * z, z ~ N(0, 1), then clips to [low, high]"""
    mean: float
    std: float
    low: float
    high: float

    def spec(self):
        """(corruptor kind, p0, p1, low, high) as b2s_obs_mod takes them"""
        return CORRUPT_GAUSSIAN, self.mean, self.std, self.low, self.high


@dataclass(frozen=True)
class UniformNoiseCorruptor:
    """adds min_noise + (max_noise - min_noise) * u, u ~ U[0, 1), then clips to [low, high]"""
    min_noise: float
    max_noise: float
    low: float
    high: float

    def spec(self):
        return CORRUPT_UNIFORM, self.min_noise, self.max_noise, self.low, self.high


def create_gaussian_noise_corruptor(mean=0.0, std=0.0, low=-math.inf, high=math.inf):
    """Gaussian noise with mean `mean` and standard deviation `std`, clipped to [low, high]"""
    mean, std, low, high = float(mean), float(std), float(low), float(high)
    if not (math.isfinite(mean) and math.isfinite(std)) or std < 0:
        raise ValueError("gaussian corruptor: mean and std must be finite and std >= 0 (mean {}, std {})".format(mean, std))
    _check_bounds(low, high)
    return GaussianNoiseCorruptor(mean, std, low, high)


def create_uniform_noise_corruptor(min_noise, max_noise, low=-math.inf, high=math.inf):
    """Uniform noise in [min_noise, max_noise), clipped to [low, high]"""
    min_noise, max_noise, low, high = float(min_noise), float(max_noise), float(low), float(high)
    if not (math.isfinite(min_noise) and math.isfinite(max_noise)) or max_noise < min_noise:
        raise ValueError("uniform corruptor: min_noise and max_noise must be finite and max_noise >= min_noise ({}, {})".format(
            min_noise, max_noise))
    _check_bounds(low, high)
    return UniformNoiseCorruptor(min_noise, max_noise, low, high)


create_gaussian_noise_corrupter = create_gaussian_noise_corruptor
create_uniform_noise_corrupter = create_uniform_noise_corruptor
