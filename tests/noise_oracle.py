"""NumPy replica of the rollout's observation and actuation noise (csrc/philox.cuh, csrc/noise.cu; TEST INFRASTRUCTURE
ONLY): Philox4x64-10 on uint64 arrays, the fp64 Box-Muller transform and x + sigma z in fp32.
numpy.random.Philox is the independent check of the generator: it increments its counter before each block, so
Philox(counter=c, key=k).random_raw(4) == philox(c + [1, 0, 0, 0], k)."""
from __future__ import annotations

import numpy as np

M0, M1 = np.uint64(0xD2E7470EE14C6C93), np.uint64(0xCA5A826395121157)
W0, W1 = np.uint64(0x9E3779B97F4A7C15), np.uint64(0xBB67AE8584CAA73B)
STATE, LIDAR, ACTION = 0, 1, 2
_LO = np.uint64(0xFFFFFFFF)
_S32 = np.uint64(32)


def _mulhilo(a: np.uint64, b: np.ndarray):
    """(high, low) 64-bit words of the 128-bit product a * b (b an array), from 32-bit halves."""
    a_lo, a_hi = a & _LO, a >> _S32
    b_lo, b_hi = b & _LO, b >> _S32
    ll, lh, hl, hh = a_lo * b_lo, a_lo * b_hi, a_hi * b_lo, a_hi * b_hi
    mid = (ll >> _S32) + (lh & _LO) + (hl & _LO)
    hi = hh + (lh >> _S32) + (hl >> _S32) + (mid >> _S32)
    return hi, a * b


def philox(counters, key) -> np.ndarray:
    """Philox4x64-10 of counters [..., 4] under key (k0, k1) -> words [..., 4] (uint64)."""
    c = np.asarray(counters, dtype=np.uint64)
    c0, c1, c2, c3 = (c[..., i].copy() for i in range(4))
    k0, k1 = np.uint64(key[0]), np.uint64(key[1])
    with np.errstate(over="ignore"):
        for r in range(10):
            if r:
                k0, k1 = k0 + W0, k1 + W1
            hi0, lo0 = _mulhilo(M0, c0)
            hi1, lo1 = _mulhilo(M1, c2)
            c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
    return np.stack([c0, c1, c2, c3], axis=-1)


def box_muller(words: np.ndarray) -> np.ndarray:
    """fp64 Box-Muller of words [..., 4]: z0, z1 from (u0, u1), z2, z3 from (u2, u3); returns fp64 [..., 4]."""
    u = ((words >> np.uint64(11)).astype(np.float64) + 0.5) * 2.0 ** -53
    out = np.empty(u.shape, dtype=np.float64)
    for p in range(2):
        rad = np.sqrt(-2.0 * np.log(u[..., 2 * p]))
        ang = 6.283185307179586 * u[..., 2 * p + 1]
        out[..., 2 * p] = rad * np.cos(ang)
        out[..., 2 * p + 1] = rad * np.sin(ang)
    return out


def normals(seed: int, kind: int, counters) -> np.ndarray:
    """The fp32 z of counters [..., 4] under key (seed, kind)."""
    return box_muller(philox(counters, (seed, kind))).astype(np.float32)


def component_z(seed: int, kind: int, t: int, env_ids, n_agents: int, n_comp: int) -> np.ndarray:
    """z of every component of every agent: [len(env_ids), n_agents, n_comp] fp32 (block j = components 4j .. 4j + 3)."""
    env_ids = np.asarray(env_ids, dtype=np.uint64)
    nb = (n_comp + 3) // 4
    c = np.zeros((len(env_ids), n_agents, nb, 4), dtype=np.uint64)
    c[..., 0] = t
    c[..., 1] = env_ids[:, None, None]
    c[..., 2] = np.arange(n_agents, dtype=np.uint64)[None, :, None]
    c[..., 3] = np.arange(nb, dtype=np.uint64)[None, None, :]
    return normals(seed, kind, c).reshape(len(env_ids), n_agents, nb * 4)[..., :n_comp]


def perturb(x: np.ndarray, sigma, z: np.ndarray) -> np.ndarray:
    """x + sigma z in fp32 with sigma broadcast over the last axis; components with sigma 0 are copied."""
    x = np.asarray(x, dtype=np.float32)
    s = np.broadcast_to(np.asarray(sigma, dtype=np.float32), x.shape)
    return np.where(s == 0, x, x + s * z.reshape(x.shape).astype(np.float32)).astype(np.float32)


def observe(seed: int, t: int, env_ids, agent: np.ndarray, hits: np.ndarray, state_sigma, lidar_sigma: float,
            comm_radius: float):
    """(x_hat, h_hat) of true agent [G, N, sd] and hits [G, N, R, pd]; no-hit sentinels (farther than 2 comm_radius
    from the agent, fp32 distance) are copied."""
    G, N, sd = agent.shape
    R, pd = hits.shape[2], hits.shape[3]
    x_hat = perturb(agent, state_sigma, component_z(seed, STATE, t, env_ids, N, sd))
    zl = component_z(seed, LIDAR, t, env_ids, N, R * pd).reshape(G, N, R, pd)
    d = agent[:, :, None, :pd].astype(np.float32) - hits.astype(np.float32)
    dsq = np.zeros(d.shape[:-1], dtype=np.float32)
    for q in range(pd):
        dsq = (dsq + d[..., q] * d[..., q]).astype(np.float32)
    far = np.float32(2.0) * np.float32(comm_radius)
    sig = np.where((dsq > far * far)[..., None], np.float32(0), np.float32(lidar_sigma))
    h_hat = perturb(hits, sig, zl)
    return x_hat, h_hat


def act_noise(seed: int, t: int, env_ids, action: np.ndarray, action_sigma) -> np.ndarray:
    G, N, nu = action.shape
    return perturb(action, action_sigma, component_z(seed, ACTION, t, env_ids, N, nu))
