// noise.cu -- observation and actuation noise of the step-by-step rollout: x_hat = x + sigma_x z on every agent state,
// h_hat = h + sigma_l z on every LiDAR hit position, a = a_cmd + sigma_u z on every applied action (DESIGN.md 4.11).
// z are standard normals of Philox4x64-10 (philox.cuh): key (seed, kind), counter (t, env_offset + g, agent, block);
// block j holds components 4j .. 4j + 3 of the agent's flattened state / [R, pd] LiDAR / action vector.  Nothing here
// depends on the batch size, so an episode's draws are the same in every batch it runs in.
// The seed and the sigmas are read from a device buffer (GCBF_NOISE_FLOATS), so new values need no new launch
// parameters; t and env_offset are launch parameters.
#include <algorithm>

#include "common.cuh"
#include "philox.cuh"

namespace gcbf {

// the noise buffer: words 0-1 the uint64 seed, then sigma_x[6], sigma_l, sigma_u[3]
constexpr int NOISE_SIGMA_X = 2, NOISE_SIGMA_L = 8, NOISE_SIGMA_U = 9;
enum { NOISE_STATE = 0, NOISE_LIDAR = 1, NOISE_ACTION = 2 };

__device__ __forceinline__ uint64_t noise_seed(const float* noise) {
    return *reinterpret_cast<const uint64_t*>(noise);
}

// x + sigma z for component c of the agent's vector; sigma == 0 copies x (so -0.0 stays -0.0)
__device__ __forceinline__ float perturb(float x, float sigma, uint64_t seed, int kind, int64_t t, int64_t env,
                                         int agent, int64_t c) {
    if (sigma == 0.f) return x;
    float z[4];
    normal4(seed, (uint64_t)kind, (uint64_t)t, (uint64_t)env, (uint64_t)agent, (uint64_t)(c >> 2), z);
    return x + sigma * z[c & 3];
}

// One thread per component: the A sd state components, then the A R pd LiDAR components.  A hit farther than twice
// the ray length (comm_radius) from its agent's true position is the no-hit sentinel (the 1e6-range point) and is
// copied unchanged.
__global__ void perturb_observation_kernel(int N, int sd, int R, int pd, float far_sq, const float* __restrict__ noise,
                                           int64_t t, int64_t env_offset, const float* __restrict__ agent,
                                           const float* __restrict__ hits, float* __restrict__ obs_agent,
                                           float* __restrict__ obs_hits, int64_t n_state, int64_t n_total) {
    const uint64_t seed = noise_seed(noise);
    for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < n_total; k += (int64_t)gridDim.x * blockDim.x) {
        if (k < n_state) {
            const int64_t a = k / sd;
            const int c = (int)(k - a * sd);
            obs_agent[k] = perturb(agent[k], noise[NOISE_SIGMA_X + c], seed, NOISE_STATE, t, env_offset + a / N,
                                   (int)(a % N), c);
            continue;
        }
        const int64_t kh = k - n_state, a = kh / (R * pd);
        const int c = (int)(kh - a * R * pd);
        const float* h = hits + kh - c % pd;
        const float* p = agent + a * sd;
        float dsq = 0.f;
        for (int q = 0; q < pd; ++q) dsq += (p[q] - h[q]) * (p[q] - h[q]);
        const float sigma = dsq > far_sq ? 0.f : noise[NOISE_SIGMA_L];
        obs_hits[kh] = perturb(hits[kh], sigma, seed, NOISE_LIDAR, t, env_offset + a / N, (int)(a % N), c);
    }
}

__global__ void perturb_action_kernel(int N, int nu, const float* __restrict__ noise, int64_t t, int64_t env_offset,
                                      float* __restrict__ action, int64_t n_total) {
    const uint64_t seed = noise_seed(noise);
    for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < n_total; k += (int64_t)gridDim.x * blockDim.x) {
        const int64_t a = k / nu;
        const int c = (int)(k - a * nu);
        action[k] = perturb(action[k], noise[NOISE_SIGMA_U + c], seed, NOISE_ACTION, t, env_offset + a / N,
                            (int)(a % N), c);
    }
}

__global__ void normal_draws_kernel(uint64_t seed, uint64_t kind, const uint64_t* __restrict__ counters, int64_t n,
                                    float* __restrict__ out) {
    for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x) {
        const uint64_t* c = counters + 4 * k;
        uint64_t w[4];
        philox4x64_10(c[0], c[1], c[2], c[3], seed, kind, w);
        float z[4];
        box_muller4(w, z);
        for (int q = 0; q < 4; ++q) out[4 * k + q] = z[q];
    }
}

static int grid_for(int64_t n) {
    return (int)std::min<int64_t>((n + 255) / 256, (int64_t)sm_count() * 16);
}

static int32_t check_noise_desc(const gcbf_env_desc* d, const char* fn) {
    GCBF_REQUIRE(d, "%s: desc is NULL", fn);
    GCBF_REQUIRE(d->env_kind >= 0 && d->env_kind <= 3 && d->n_graphs > 0 && d->n_agents > 0 && d->n_hits > 0,
                 "%s: bad descriptor (env_kind %d, n_graphs %d, n_agents %d, n_hits %d)", fn, d->env_kind, d->n_graphs,
                 d->n_agents, d->n_hits);
    GCBF_REQUIRE((int64_t)d->n_graphs * d->n_agents < (int64_t)1 << 30, "%s: too many agents", fn);
    return 0;
}

}  // namespace gcbf

using namespace gcbf;

extern "C" __attribute__((visibility("default"))) int32_t gcbf_perturb_observation(
    const gcbf_env_desc* desc, const float* noise, int64_t t, int64_t env_offset, const float* agent, const float* hits,
    float* obs_agent, float* obs_hits, void* stream) {
    if (int32_t rc = check_noise_desc(desc, "gcbf_perturb_observation")) return rc;
    GCBF_REQUIRE(noise && agent && hits && obs_agent && obs_hits, "gcbf_perturb_observation: NULL pointer argument");
    GCBF_REQUIRE(((uintptr_t)noise & 7) == 0, "gcbf_perturb_observation: noise must be 8-byte aligned");
    GCBF_REQUIRE(obs_agent != agent && obs_hits != hits, "gcbf_perturb_observation: the observation must not alias the "
                                                          "true state");
    GCBF_REQUIRE(t >= 0 && env_offset >= 0, "gcbf_perturb_observation: t (%lld) and env_offset (%lld) must be >= 0",
                 (long long)t, (long long)env_offset);
    const int sd = env_sd(desc->env_kind), pd = env_pd(desc->env_kind), R = desc->n_hits;
    const int64_t A = (int64_t)desc->n_graphs * desc->n_agents, n_state = A * sd, n_total = n_state + A * R * pd;
    const float far = 2.f * desc->comm_radius;
    perturb_observation_kernel<<<grid_for(n_total), 256, 0, (cudaStream_t)stream>>>(
        desc->n_agents, sd, R, pd, far * far, noise, t, env_offset, agent, hits, obs_agent, obs_hits, n_state, n_total);
    count_launch();
    return check_launch("perturb_observation_kernel");
}

extern "C" __attribute__((visibility("default"))) int32_t gcbf_perturb_action(const gcbf_env_desc* desc,
                                                                              const float* noise, int64_t t,
                                                                              int64_t env_offset, float* action_inout,
                                                                              void* stream) {
    if (int32_t rc = check_noise_desc(desc, "gcbf_perturb_action")) return rc;
    GCBF_REQUIRE(noise && action_inout, "gcbf_perturb_action: NULL pointer argument");
    GCBF_REQUIRE(((uintptr_t)noise & 7) == 0, "gcbf_perturb_action: noise must be 8-byte aligned");
    GCBF_REQUIRE(t >= 0 && env_offset >= 0, "gcbf_perturb_action: t (%lld) and env_offset (%lld) must be >= 0",
                 (long long)t, (long long)env_offset);
    const int nu = env_nu(desc->env_kind);
    const int64_t n_total = (int64_t)desc->n_graphs * desc->n_agents * nu;
    perturb_action_kernel<<<grid_for(n_total), 256, 0, (cudaStream_t)stream>>>(desc->n_agents, nu, noise, t,
                                                                                env_offset, action_inout, n_total);
    count_launch();
    return check_launch("perturb_action_kernel");
}

extern "C" __attribute__((visibility("default"))) int32_t gcbf_normal_draws(uint64_t seed, int32_t kind,
                                                                            const uint64_t* counters, int64_t n,
                                                                            float* out, void* stream) {
    GCBF_REQUIRE(kind >= 0 && kind <= 2, "gcbf_normal_draws: kind %d outside [0, 2]", kind);
    GCBF_REQUIRE(n >= 0 && n < (int64_t)1 << 40, "gcbf_normal_draws: bad count %lld", (long long)n);
    if (n == 0) return 0;
    GCBF_REQUIRE(counters && out, "gcbf_normal_draws: NULL pointer argument");
    normal_draws_kernel<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(seed, (uint64_t)kind, counters, n, out);
    count_launch();
    return check_launch("normal_draws_kernel");
}
