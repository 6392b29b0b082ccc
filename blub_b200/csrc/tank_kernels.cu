// tank_kernels.cu -- moving tanks (DESIGN.md §8 "Moving tanks").  Not in the reference, whose tank is always at rest.
//
// The liquid is simulated in the tank's frame.  The host rules below turn a frame (R, A, omega, alpha, pivot) into the float32 constants of one
// step: g_eff = R^T (g - A) replaces the step's gravity, and while the frame rotates tank_frame_kernel applies the rest of the frame's inertial
// forces to every live particle in stage 0, before P2G.  Its rows hold (grad v_c, v_c) per component c; the kernel
//   - rotates them by Q = Rot(omega^, -2 |omega| dt), the exact solution of the Coriolis equation dv/dt = -2 omega x v over one step, and
//   - adds the position-dependent force K r = dt (|omega|^2 r - omega (omega . r) - alpha x r), r = x - pivot: K[c] to grad v_c (the force
//     field's gradient, so that APIC's linear field stays consistent) and K[c] . r to v_c.
// Every product and sum is rounded on its own in a fixed order (__fmul_rn / __fadd_rn / __fsub_rn, no contraction), so that a NumPy
// restatement reproduces it bit for bit.  It reads 3 x 16 B of rows and 16 B of position and writes 3 x 16 B: 112 B per particle.
#include <algorithm>
#include <cmath>

#include "blub_core.hpp"

namespace blub {

namespace {

constexpr int PT = 256;

inline int blocks_for(int64_t n, int per_block) { return (int)((n + per_block - 1) / per_block); }

// n: params->num_particles in device-count mode (device_count != 0), else n_host.  The position's fourth word (the tag) is never used.
__global__ void __launch_bounds__(PT) tank_frame_kernel(const StepParams *__restrict__ params, int device_count, uint32_t n_host,
                                                        const float4 *__restrict__ pos, float4 *__restrict__ rx, float4 *__restrict__ ry,
                                                        float4 *__restrict__ rz) {
    const uint32_t n = device_count ? params->num_particles : n_host;
    float q[9], k[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) {
        q[i] = params->tank_q[i];
        k[i] = params->tank_k[i];
    }
    const float p0 = params->tank_pivot[0], p1 = params->tank_pivot[1], p2 = params->tank_pivot[2];
    for (uint32_t i = blockIdx.x * PT + threadIdx.x; i < n; i += gridDim.x * PT) {
        // streaming loads and stores: every word is touched once per step
        const float4 x = __ldcs(pos + i);
        const float4 a = __ldcs(rx + i), b = __ldcs(ry + i), c = __ldcs(rz + i);
        const float r0 = __fsub_rn(x.x, p0), r1 = __fsub_rn(x.y, p1), r2 = __fsub_rn(x.z, p2);
        float4 out[3];
#pragma unroll
        for (int row = 0; row < 3; ++row) {
            const float q0 = q[3 * row], q1 = q[3 * row + 1], q2 = q[3 * row + 2];
            const float k0 = k[3 * row], k1 = k[3 * row + 1], k2 = k[3 * row + 2];
            // row'_c = Q[c][0] row_0 + Q[c][1] row_1 + Q[c][2] row_2, then the force: .xyz += K[c], .w += K[c] . r
            const float gx = __fadd_rn(__fadd_rn(__fmul_rn(q0, a.x), __fmul_rn(q1, b.x)), __fmul_rn(q2, c.x));
            const float gy = __fadd_rn(__fadd_rn(__fmul_rn(q0, a.y), __fmul_rn(q1, b.y)), __fmul_rn(q2, c.y));
            const float gz = __fadd_rn(__fadd_rn(__fmul_rn(q0, a.z), __fmul_rn(q1, b.z)), __fmul_rn(q2, c.z));
            const float v = __fadd_rn(__fadd_rn(__fmul_rn(q0, a.w), __fmul_rn(q1, b.w)), __fmul_rn(q2, c.w));
            const float f = __fadd_rn(__fadd_rn(__fmul_rn(k0, r0), __fmul_rn(k1, r1)), __fmul_rn(k2, r2));
            out[row] = make_float4(__fadd_rn(gx, k0), __fadd_rn(gy, k1), __fadd_rn(gz, k2), __fadd_rn(v, f));
        }
        __stcs(rx + i, out[0]);
        __stcs(ry + i, out[1]);
        __stcs(rz + i, out[2]);
    }
}

bool finite_all(const double *v, int n) {
    for (int i = 0; i < n; ++i)
        if (!std::isfinite(v[i])) return false;
    return true;
}

double norm3(const double v[3]) { return std::sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]); }

void check_unit(const double v[3], const char *what) {
    if (!finite_all(v, 3) || std::fabs(norm3(v) - 1.0) > 1e-6) throw std::invalid_argument(std::string("tank motion: ") + what + " is not a unit vector");
}

// Rot(n, theta) by Rodrigues' formula, row major (n a unit vector)
void rotation_about(const double n[3], double theta, double out[9]) {
    const double c = std::cos(theta), s = std::sin(theta), t = 1.0 - c;
    out[0] = c + t * n[0] * n[0];        out[1] = t * n[0] * n[1] - s * n[2]; out[2] = t * n[0] * n[2] + s * n[1];
    out[3] = t * n[1] * n[0] + s * n[2]; out[4] = c + t * n[1] * n[1];        out[5] = t * n[1] * n[2] - s * n[0];
    out[6] = t * n[2] * n[0] - s * n[1]; out[7] = t * n[2] * n[1] + s * n[0]; out[8] = c + t * n[2] * n[2];
}

} // namespace

void launch_tank_frame(cudaStream_t st, const StepParams *params, bool device_count, uint32_t n_host, uint32_t np_upper, const float4 *pos,
                       float4 *const row[3]) {
    if (np_upper == 0) return;
    // 8 blocks of 256 threads per SM, a grid-stride loop over the rest
    BLUB_LAUNCH(tank_frame_kernel, std::min(blocks_for(np_upper, PT), device_sm_count() * 8), PT, 0, st, params, device_count ? 1 : 0, n_host, pos,
                row[0], row[1], row[2]);
}

void check_tank_frame(const BlubTankFrame &f) {
    if (!finite_all(f.rotation, 9) || !finite_all(f.acceleration, 3) || !finite_all(f.angular_velocity, 3) || !finite_all(f.angular_acceleration, 3) ||
        !finite_all(f.pivot, 3))
        throw std::invalid_argument("tank frame: a value is not finite");
    const double *R = f.rotation;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            const double d = R[i] * R[j] + R[3 + i] * R[3 + j] + R[6 + i] * R[6 + j]; // (R^T R)_ij
            if (std::fabs(d - (i == j ? 1.0 : 0.0)) > 1e-6) throw std::invalid_argument("tank frame: the rotation is not orthonormal to 1e-6");
        }
    const double det = R[0] * (R[4] * R[8] - R[5] * R[7]) - R[1] * (R[3] * R[8] - R[5] * R[6]) + R[2] * (R[3] * R[7] - R[4] * R[6]);
    if (std::fabs(det - 1.0) > 1e-6) throw std::invalid_argument("tank frame: the rotation's determinant is not +1 to 1e-6");
}

bool tank_frame_rotates(const BlubTankFrame &f) {
    for (int c = 0; c < 3; ++c)
        if (f.angular_velocity[c] != 0.0 || f.angular_acceleration[c] != 0.0) return true;
    return false;
}

BlubTankFrame tank_frame_at(const BlubTankMotion &m, double t) {
    if (!std::isfinite(t)) throw std::invalid_argument("tank motion: the time is not finite");
    if (m.num_translations > BLUB_TANK_TRANSLATIONS_MAX) throw std::invalid_argument("tank motion: at most 4 translations");
    if (m.reserved != 0u) throw std::invalid_argument("tank motion: reserved must be 0");
    if (!finite_all(m.pivot, 3)) throw std::invalid_argument("tank motion: the pivot is not finite");
    BlubTankFrame f{};
    for (uint32_t i = 0; i < m.num_translations; ++i) {
        const BlubTankTranslation &tr = m.translations[i];
        check_unit(tr.direction, "a translation direction");
        if (!std::isfinite(tr.amplitude) || !std::isfinite(tr.frequency) || !std::isfinite(tr.phase) || tr.frequency < 0.0)
            throw std::invalid_argument("tank motion: a translation's amplitude, frequency or phase is not finite, or its frequency is negative");
        const double w = 2.0 * M_PI * tr.frequency;
        const double a = -tr.amplitude * w * w * std::sin(w * t + tr.phase); // d^2/dt^2 of amplitude sin(w t + phase)
        for (int c = 0; c < 3; ++c) f.acceleration[c] += a * tr.direction[c];
    }
    check_unit(m.axis, "the rotation axis");
    if (!std::isfinite(m.amplitude) || !std::isfinite(m.frequency) || !std::isfinite(m.phase) || !std::isfinite(m.rate) || m.frequency < 0.0)
        throw std::invalid_argument("tank motion: the rotation's amplitude, frequency, phase or rate is not finite, or its frequency is negative");
    const double w = 2.0 * M_PI * m.frequency, arg = w * t + m.phase;
    const double theta = m.amplitude * std::sin(arg) + m.rate * t;
    const double theta1 = m.amplitude * w * std::cos(arg) + m.rate;
    const double theta2 = -m.amplitude * w * w * std::sin(arg);
    rotation_about(m.axis, theta, f.rotation);
    for (int c = 0; c < 3; ++c) {
        f.angular_velocity[c] = theta1 * m.axis[c];
        f.angular_acceleration[c] = theta2 * m.axis[c];
        f.pivot[c] = m.pivot[c];
    }
    return f;
}

BlubTankStepConstants tank_step_constants(const BlubTankFrame &f, const float g[3], float dt) {
    check_tank_frame(f);
    if (!std::isfinite(g[0]) || !std::isfinite(g[1]) || !std::isfinite(g[2])) throw std::invalid_argument("tank step constants: gravity is not finite");
    if (!(dt > 0.0f) || !std::isfinite(dt)) throw std::invalid_argument("tank step constants: dt must be finite and above 0");
    BlubTankStepConstants out{};
    const double *R = f.rotation, *w = f.angular_velocity, *al = f.angular_acceleration;
    const double h = (double)dt;
    double d[3];
    for (int c = 0; c < 3; ++c) d[c] = (double)g[c] - f.acceleration[c];
    for (int c = 0; c < 3; ++c) out.gravity[c] = (float)(R[c] * d[0] + R[3 + c] * d[1] + R[6 + c] * d[2]); // (R^T d)_c
    const double wn = norm3(w);
    double Q[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    if (wn > 0.0) {
        const double n[3] = {w[0] / wn, w[1] / wn, w[2] / wn};
        rotation_about(n, -2.0 * wn * h, Q);
    }
    const double w2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2];
    // [alpha]x r = alpha x r
    const double ax[9] = {0.0, -al[2], al[1], al[2], 0.0, -al[0], -al[1], al[0], 0.0};
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            out.coriolis[3 * i + j] = (float)Q[3 * i + j];
            out.force[3 * i + j] = (float)(h * ((i == j ? w2 : 0.0) - w[i] * w[j] - ax[3 * i + j]));
        }
    for (int c = 0; c < 3; ++c) out.pivot[c] = (float)f.pivot[c];
    out.rotating = tank_frame_rotates(f) ? 1 : 0;
    return out;
}

uint64_t tank_cfl_substep_ns(uint64_t remaining_ns, const float max_velocity[3], const float gravity_grid[3], const BlubTankFrame *frame,
                             const uint32_t dim[3], const BlubTimeStepping &ts) {
    if (!frame) return cfl_substep_ns(remaining_ns, max_velocity, gravity_grid, ts);
    check_time_stepping(ts);
    if (remaining_ns == 0) throw std::invalid_argument("cfl substep: remaining_ns must be above 0");
    // g_eff does not depend on dt: any positive step gives the same float32 gravity
    const BlubTankStepConstants k = tank_step_constants(*frame, gravity_grid, 1.0f);
    double r_max = 0.0;
    for (int corner = 0; corner < 8; ++corner) {
        double r2 = 0.0;
        for (int c = 0; c < 3; ++c) {
            const double e = ((corner >> c) & 1 ? (double)dim[c] : 0.0) - frame->pivot[c];
            r2 += e * e;
        }
        r_max = std::max(r_max, std::sqrt(r2));
    }
    const double *w = frame->angular_velocity;
    const double geff = std::sqrt((double)k.gravity[0] * k.gravity[0] + (double)k.gravity[1] * k.gravity[1] + (double)k.gravity[2] * k.gravity[2]);
    const float g_bound[3] = {(float)(geff + (w[0] * w[0] + w[1] * w[1] + w[2] * w[2] + norm3(frame->angular_acceleration)) * r_max), 0.0f, 0.0f};
    float v[3] = {max_velocity[0], max_velocity[1], max_velocity[2]};
    if (w[0] != 0.0 || w[1] != 0.0 || w[2] != 0.0) {
        v[0] = (float)std::sqrt((double)v[0] * v[0] + (double)v[1] * v[1] + (double)v[2] * v[2]); // non-finite stays non-finite
        v[1] = v[2] = 0.0f;
    }
    return cfl_substep_ns(remaining_ns, v, g_bound, ts);
}

} // namespace blub
