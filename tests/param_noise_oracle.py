"""NumPy restatement of adaptive parameter-space noise (DESIGN.md §3 "Parameter-space noise"): a vectorised Philox4x32-10
uniform53, the perturbation of the actor's logical parameters, the fp64 policy distance and baselines' sigma rule."""
import numpy as np

PERTURB_COUNTER_BASE = (1 << 63) + (1 << 62)      # perturbation j draws with counter 2^63 + 2^62 + j
_M0, _M1, _MASK = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57), np.uint64(0xFFFFFFFF)


def uniform53(seed, counter, lanes):
    """Philox::uniform53(seed, counter, lane) (csrc/common.cuh) for an array of 32-bit lanes at once."""
    lanes = np.asarray(lanes, dtype=np.uint64)
    c0 = np.full(lanes.shape, counter & 0xFFFFFFFF, np.uint64)
    c1 = np.full(lanes.shape, (counter >> 32) & 0xFFFFFFFF, np.uint64)
    c2 = lanes & _MASK
    c3 = np.full(lanes.shape, 0x9E3779B9, np.uint64)
    k0, k1 = seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF
    for _ in range(10):
        p0, p1 = _M0 * c0, _M1 * c2                    # 32 x 32 -> 64-bit products, exact in uint64
        c0, c1, c2, c3 = (((p1 >> np.uint64(32)) ^ c1 ^ np.uint64(k0)) & _MASK, p1 & _MASK,
                          ((p0 >> np.uint64(32)) ^ c3 ^ np.uint64(k1)) & _MASK, p0 & _MASK)
        k0, k1 = (k0 + 0x9E3779B9) & 0xFFFFFFFF, (k1 + 0xBB67AE85) & 0xFFFFFFFF
    a, b = (c0 >> np.uint64(5)).astype(np.float64), (c1 >> np.uint64(6)).astype(np.float64)
    return (a * 67108864.0 + b) * (1.0 / 9007199254740992.0)


def standard_normal(seed, counter, n):
    """z_i = sqrt(-2 log(1 - u1)) * cos(2 pi u2), u1 / u2 = uniform53(seed, counter, 2i / 2i + 1), i < n."""
    i = np.arange(n, dtype=np.uint64)
    u1 = uniform53(seed, counter, 2 * i)
    u2 = uniform53(seed, counter, 2 * i + 1)
    return np.sqrt(-2.0 * np.log(1.0 - u1)) * np.cos(2.0 * np.pi * u2)


def perturb(params, sigma, seed, j):
    """Perturbation j of the logical parameter vector `params` (fp32, torch.cat of the flattened parameters):
    float32(float64(p) + sigma * z)."""
    p = np.asarray(params, dtype=np.float32).reshape(-1)
    z = standard_normal(seed, PERTURB_COUNTER_BASE + j, p.size)
    return (p.astype(np.float64) + np.float64(sigma) * z).astype(np.float32)


def distance(a, a_perturbed):
    """d = sqrt(sum (f64(a_perturbed) - f64(a))^2 / n) in fp64."""
    diff = np.asarray(a_perturbed, np.float32).astype(np.float64) - np.asarray(a, np.float32).astype(np.float64)
    return float(np.sqrt(np.sum(diff * diff) / diff.size))


def adapt(sigma, d, desired, coef):
    """baselines' AdaptiveParamNoiseSpec.adapt: shrink when the distance exceeds the target, grow otherwise (ties grow)."""
    return float(np.float64(sigma) / np.float64(coef)) if d > desired else float(np.float64(sigma) * np.float64(coef))


def actor_forward(params, s):
    """The actor in fp64 on numpy parameters {name: array} (fc1 -> relu -> fc2 -> fc2_2 -> relu -> fc3 -> tanh)."""
    h = np.asarray(s, np.float64)
    for name, act in (("fc1", "relu"), ("fc2", None), ("fc2_2", "relu"), ("fc3", "tanh")):
        h = h @ np.asarray(params[name + ".weight"], np.float64).T + np.asarray(params[name + ".bias"], np.float64)
        h = np.maximum(h, 0.0) if act == "relu" else np.tanh(h) if act == "tanh" else h
    return h
