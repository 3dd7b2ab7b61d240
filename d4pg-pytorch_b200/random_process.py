"""Exploration-noise processes constructed by DDPG.__init__ (ddpg.py:75).  Actor-side helpers,
outside the learner hot path; kept so `ddpg.noise.sample()` / `.reset()` callers keep working
(reference: random_process.py:4-45)."""
import numpy as np


class _DecayingNoise(object):
    min_epsilon = 0.01

    def _decayed(self, rate, it):
        return self.min_epsilon + (1.0 - self.min_epsilon) * np.exp(-rate * it)


class GaussianNoise(_DecayingNoise):
    def __init__(self, dimension, num_epochs, mu=0.0, var=1):
        self.mu, self.var, self.dimension = mu, var, dimension
        self.epochs, self.num_epochs = 0, num_epochs
        self.epsilon = 0.3
        self.decay_rate = 5.0 / num_epochs
        self.iter = 0

    def sample(self):
        return self.epsilon * np.random.normal(self.mu, self.var, size=self.dimension)

    def reset(self):
        self.epsilon = self._decayed(self.decay_rate, self.iter)


class OrnsteinUhlenbeckProcess(_DecayingNoise):
    def __init__(self, dimension, num_steps, theta=0.25, mu=0.0, sigma=0.05, dt=0.01):
        self.theta, self.mu, self.sigma, self.dt = theta, mu, sigma, dt
        self.dimension, self.num_steps = dimension, num_steps
        self.x = np.zeros((dimension,))
        self.iter = 0
        self.epsilon = 1.0
        self.decay_rate = 5.0 / num_steps

    def sample(self):
        drift = self.theta * (self.mu - self.x) * self.dt
        diffusion = self.sigma * np.sqrt(self.dt) * np.random.normal(size=self.dimension)
        self.x = self.x + drift + diffusion
        return self.epsilon * self.x

    def reset(self):
        self.x = np.zeros_like(self.x)
        self.iter += 1
        self.epsilon = self._decayed(self.decay_rate, self.iter)


class AdaptiveParamNoiseSpec(object):
    """Adaptive parameter-space noise (Plappert et al. 2018; baselines' AdaptiveParamNoiseSpec, same defaults), selected
    with DDPG(param_noise=spec).  The actor's parameters get Gaussian noise of std dev sigma, which starts at
    `initial_stddev`; DDPG.adapt_param_noise divides sigma by `adoption_coefficient` when the perturbed actor's actions
    lie more than `desired_action_stddev` (RMS) from the actor's, and multiplies it otherwise.  sigma lives on the
    device (DDPG.param_noise_state); the attributes here are read, and checked, at every use."""

    def __init__(self, initial_stddev=0.1, desired_action_stddev=0.1, adoption_coefficient=1.01):
        self.initial_stddev = initial_stddev
        self.desired_action_stddev = desired_action_stddev
        self.adoption_coefficient = adoption_coefficient
        self.check()

    def check(self):
        """(initial_stddev, desired_action_stddev, adoption_coefficient) as floats; ValueError when one is out of range."""
        out = []
        for name, ok, what in (("initial_stddev", lambda v: v >= 0.0, ">= 0"),
                               ("desired_action_stddev", lambda v: v > 0.0, "> 0"),
                               ("adoption_coefficient", lambda v: v > 1.0, "> 1")):
            raw = getattr(self, name)
            try:
                v = float(raw)
            except (TypeError, ValueError):
                raise ValueError("AdaptiveParamNoiseSpec.%s must be a number, got %r" % (name, raw))
            if not (np.isfinite(v) and ok(v)):
                raise ValueError("AdaptiveParamNoiseSpec.%s must be finite and %s, got %r" % (name, what, raw))
            out.append(v)
        return tuple(out)

    def __repr__(self):
        return "AdaptiveParamNoiseSpec(initial_stddev=%r, desired_action_stddev=%r, adoption_coefficient=%r)" % (
            self.initial_stddev, self.desired_action_stddev, self.adoption_coefficient)
