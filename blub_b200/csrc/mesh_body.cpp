// mesh_body.cpp -- host side of the triangle-mesh bodies (DESIGN.md §8 "Mesh bodies").  Not in the reference.
//
// Checks a closed mesh, computes its mass properties in float64 by the divergence theorem over signed tetrahedra, finds the principal frame
// with a cyclic Jacobi eigensolver and re-expresses the mesh in that frame as the float32 vertices the device fills from.
#include <algorithm>
#include <cmath>
#include <stdexcept>
#include <string>
#include <unordered_map>

#include "blub_core.hpp"

namespace blub {

namespace {

void refuse(const std::string &what) { throw std::invalid_argument("mesh body: " + what); }

// eigenvalues d and eigenvectors (columns of V) of the symmetric 3 x 3 matrix A: cyclic Jacobi, pairs (0,1), (0,2), (1,2) in that order
void jacobi3(const double A_in[9], double d[3], double V[9]) {
    double A[9];
    std::copy(A_in, A_in + 9, A);
    for (int k = 0; k < 9; ++k) V[k] = k % 4 == 0 ? 1.0 : 0.0;
    const double scale = std::fabs(A[0]) + std::fabs(A[4]) + std::fabs(A[8]);
    static const int pairs[3][2] = {{0, 1}, {0, 2}, {1, 2}};
    for (int sweep = 0; sweep < 64; ++sweep) {
        const double off = std::fabs(A[1]) + std::fabs(A[2]) + std::fabs(A[5]);
        if (off <= 1e-17 * scale) break;
        for (const auto &pq : pairs) {
            const int p = pq[0], q = pq[1];
            const double apq = A[3 * p + q];
            if (apq == 0.0) continue;
            const double theta = (A[3 * q + q] - A[3 * p + p]) / (2.0 * apq);
            const double t = (theta >= 0.0 ? 1.0 : -1.0) / (std::fabs(theta) + std::sqrt(theta * theta + 1.0));
            const double c = 1.0 / std::sqrt(t * t + 1.0), s = t * c;
            for (int k = 0; k < 3; ++k) { // A <- A J
                const double akp = A[3 * k + p], akq = A[3 * k + q];
                A[3 * k + p] = c * akp - s * akq;
                A[3 * k + q] = s * akp + c * akq;
            }
            for (int k = 0; k < 3; ++k) { // A <- J^T A
                const double apk = A[3 * p + k], aqk = A[3 * q + k];
                A[3 * p + k] = c * apk - s * aqk;
                A[3 * q + k] = s * apk + c * aqk;
            }
            for (int k = 0; k < 3; ++k) { // V <- V J
                const double vkp = V[3 * k + p], vkq = V[3 * k + q];
                V[3 * k + p] = c * vkp - s * vkq;
                V[3 * k + q] = s * vkp + c * vkq;
            }
        }
    }
    for (int k = 0; k < 3; ++k) d[k] = A[4 * k];
}

// unit quaternion (w, x, y, z) of the rotation matrix R (row major), w >= 0
void quat_of(const double R[9], double q[4]) {
    const double tr = R[0] + R[4] + R[8];
    if (tr > 0.0) {
        const double s = 2.0 * std::sqrt(1.0 + tr);
        q[0] = 0.25 * s, q[1] = (R[7] - R[5]) / s, q[2] = (R[2] - R[6]) / s, q[3] = (R[3] - R[1]) / s;
    } else if (R[0] >= R[4] && R[0] >= R[8]) {
        const double s = 2.0 * std::sqrt(1.0 + R[0] - R[4] - R[8]);
        q[0] = (R[7] - R[5]) / s, q[1] = 0.25 * s, q[2] = (R[1] + R[3]) / s, q[3] = (R[2] + R[6]) / s;
    } else if (R[4] >= R[8]) {
        const double s = 2.0 * std::sqrt(1.0 + R[4] - R[0] - R[8]);
        q[0] = (R[2] - R[6]) / s, q[1] = (R[1] + R[3]) / s, q[2] = 0.25 * s, q[3] = (R[5] + R[7]) / s;
    } else {
        const double s = 2.0 * std::sqrt(1.0 + R[8] - R[0] - R[4]);
        q[0] = (R[3] - R[1]) / s, q[1] = (R[2] + R[6]) / s, q[2] = (R[5] + R[7]) / s, q[3] = 0.25 * s;
    }
    const double n = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]) * (q[0] < 0.0 ? -1.0 : 1.0);
    for (int k = 0; k < 4; ++k) q[k] /= n;
}

} // namespace

void quat_rotation_f64(const double q[4], double R[9]) {
    const double w = q[0], x = q[1], y = q[2], z = q[3];
    R[0] = 1 - 2 * (y * y + z * z), R[1] = 2 * (x * y - w * z), R[2] = 2 * (x * z + w * y);
    R[3] = 2 * (x * y + w * z), R[4] = 1 - 2 * (x * x + z * z), R[5] = 2 * (y * z - w * x);
    R[6] = 2 * (x * z - w * y), R[7] = 2 * (y * z + w * x), R[8] = 1 - 2 * (x * x + y * y);
}

BlubMeshBodyProperties mesh_body_properties(const float *positions, uint32_t num_vertices, const uint32_t *indices, uint32_t num_indices, float scale,
                                            std::vector<float> *body_vertices) {
    if (!(std::isfinite(scale) && scale > 0.0f)) refuse("the scale must be finite and > 0");
    if (num_indices == 0 || num_vertices == 0) refuse("the mesh is empty");
    if (num_indices % 3 != 0) refuse("the number of indices is not a multiple of 3");
    if (!positions || !indices) refuse("NULL positions or indices");
    if (num_vertices > (uint32_t)BLUB_MESH_BODY_MAX_VERTICES || num_indices / 3 > (uint32_t)BLUB_MESH_BODY_MAX_TRIANGLES)
        refuse("more than " + std::to_string(BLUB_MESH_BODY_MAX_VERTICES) + " vertices or " + std::to_string(BLUB_MESH_BODY_MAX_TRIANGLES) + " triangles");
    for (uint32_t k = 0; k < 3 * num_vertices; ++k)
        if (!std::isfinite(positions[k])) refuse("a position is not finite");
    // closed and consistently oriented: every directed edge exactly once, and its reverse too
    std::unordered_map<uint64_t, uint32_t> edges;
    edges.reserve((size_t)num_indices * 2);
    for (uint32_t t = 0; t < num_indices; t += 3) {
        for (int k = 0; k < 3; ++k)
            if (indices[t + k] >= num_vertices) refuse("an index is out of range");
        if (indices[t] == indices[t + 1] || indices[t + 1] == indices[t + 2] || indices[t] == indices[t + 2]) refuse("a triangle repeats a vertex");
        for (int k = 0; k < 3; ++k)
            if (++edges[(uint64_t)indices[t + k] << 32 | indices[t + (k + 1) % 3]] != 1) refuse("a directed edge occurs twice (the mesh is not consistently oriented)");
    }
    for (const auto &e : edges)
        if (!edges.count(e.first >> 32 | e.first << 32)) refuse("an edge has no reverse (the mesh is not closed)");

    BlubMeshBodyProperties out{};
    out.scale = scale;
    out.num_vertices = num_vertices;
    out.num_triangles = num_indices / 3;
    // the scaled positions about their mean, so that a mesh far from its model origin keeps its precision
    std::vector<double> p(3 * (size_t)num_vertices);
    double mean[3] = {0, 0, 0}, bmin[3] = {INFINITY, INFINITY, INFINITY}, bmax[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (uint32_t v = 0; v < num_vertices; ++v)
        for (int k = 0; k < 3; ++k) {
            const double x = (double)scale * (double)positions[3 * v + k];
            p[3 * v + k] = x;
            mean[k] += x;
            bmin[k] = std::min(bmin[k], x);
            bmax[k] = std::max(bmax[k], x);
        }
    for (int k = 0; k < 3; ++k) mean[k] /= num_vertices;
    for (uint32_t v = 0; v < num_vertices; ++v)
        for (int k = 0; k < 3; ++k) p[3 * v + k] -= mean[k];
    // signed tetrahedra (0, a, b, c): det = a . (b x c); int x dV = det (a + b + c) / 24, int x x^T dV = det (a a^T + b b^T + c c^T + s s^T) / 120
    double V6 = 0.0, S[3] = {0, 0, 0}, C[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (uint32_t t = 0; t < num_indices; t += 3) {
        const double *a = &p[3 * (size_t)indices[t]], *b = &p[3 * (size_t)indices[t + 1]], *c = &p[3 * (size_t)indices[t + 2]];
        const double det = a[0] * (b[1] * c[2] - b[2] * c[1]) + a[1] * (b[2] * c[0] - b[0] * c[2]) + a[2] * (b[0] * c[1] - b[1] * c[0]);
        const double s[3] = {a[0] + b[0] + c[0], a[1] + b[1] + c[1], a[2] + b[2] + c[2]};
        V6 += det;
        for (int i = 0; i < 3; ++i) {
            S[i] += det * s[i];
            for (int j = 0; j < 3; ++j) C[3 * i + j] += det * (a[i] * a[j] + b[i] * b[j] + c[i] * c[j] + s[i] * s[j]);
        }
    }
    const double sign = V6 < 0.0 ? -1.0 : 1.0; // inward winding: every integral changes sign
    const double V = sign * V6 / 6.0;
    const double box = (bmax[0] - bmin[0]) * (bmax[1] - bmin[1]) * (bmax[2] - bmin[2]);
    if (!(V > 1e-9 * box) || !(V > 0.0)) refuse("the mesh encloses no volume");
    double com[3], I[9];
    for (int i = 0; i < 3; ++i) com[i] = sign * S[i] / 24.0 / V;
    double Cc[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) Cc[3 * i + j] = sign * C[3 * i + j] / 120.0 - V * com[i] * com[j];
    const double trace = Cc[0] + Cc[4] + Cc[8];
    for (int i = 0; i < 9; ++i) I[i] = (i % 4 == 0 ? trace : 0.0) - Cc[i];
    out.volume = V;
    for (int k = 0; k < 3; ++k) out.centroid[k] = (com[k] + mean[k]) / (double)scale;
    std::copy(I, I + 9, out.inertia);
    // the principal frame: the model frame when the products of inertia are negligible, else Jacobi with the documented order and signs
    double d[3], Rp[9];
    const double itrace = I[0] + I[4] + I[8];
    if (std::max({std::fabs(I[1]), std::fabs(I[2]), std::fabs(I[5])}) <= 1e-9 * itrace) {
        for (int k = 0; k < 3; ++k) d[k] = I[4 * k];
        for (int k = 0; k < 9; ++k) Rp[k] = k % 4 == 0 ? 1.0 : 0.0;
    } else {
        double e[3], E[9];
        jacobi3(I, e, E);
        int order[3] = {0, 1, 2};
        std::stable_sort(order, order + 3, [&](int a, int b) { return e[a] < e[b]; }); // ascending moments
        for (int j = 0; j < 3; ++j) {
            d[j] = e[order[j]];
            int big = 0;
            for (int i = 1; i < 3; ++i)
                if (std::fabs(E[3 * i + order[j]]) > std::fabs(E[3 * big + order[j]])) big = i;
            const double s = E[3 * big + order[j]] < 0.0 ? -1.0 : 1.0; // the largest component of each axis is positive
            for (int i = 0; i < 3; ++i) Rp[3 * i + j] = s * E[3 * i + order[j]];
        }
        const double det = Rp[0] * (Rp[4] * Rp[8] - Rp[5] * Rp[7]) - Rp[1] * (Rp[3] * Rp[8] - Rp[5] * Rp[6]) + Rp[2] * (Rp[3] * Rp[7] - Rp[4] * Rp[6]);
        if (det < 0.0)
            for (int i = 0; i < 3; ++i) Rp[3 * i + 2] = -Rp[3 * i + 2]; // right-handed: the third axis gives way
    }
    std::copy(d, d + 3, out.principal_moments);
    quat_of(Rp, out.principal_rotation);
    // the body frame: v_b = R_p^T (p - com), rounded to float32 once
    std::vector<float> vb(3 * (size_t)num_vertices);
    for (int k = 0; k < 3; ++k) out.bounds_lo[k] = INFINITY, out.bounds_hi[k] = -INFINITY;
    for (uint32_t v = 0; v < num_vertices; ++v) {
        const double r[3] = {p[3 * v] - com[0], p[3 * v + 1] - com[1], p[3 * v + 2] - com[2]};
        for (int j = 0; j < 3; ++j) {
            const float x = (float)(Rp[j] * r[0] + Rp[3 + j] * r[1] + Rp[6 + j] * r[2]);
            vb[3 * (size_t)v + j] = x;
            out.bounds_lo[j] = std::min(out.bounds_lo[j], x);
            out.bounds_hi[j] = std::max(out.bounds_hi[j], x);
        }
    }
    for (int k = 0; k < 3; ++k)
        if (!(out.bounds_hi[k] - out.bounds_lo[k] >= 1.0f)) refuse("the body-frame bounding box is thinner than 1 cell");
    out.mass = (float)V;
    for (int k = 0; k < 3; ++k) out.moments[k] = (float)d[k];
    if (body_vertices) *body_vertices = std::move(vb);
    return out;
}

MeshBodyHost make_mesh_body(const uint32_t dim[3], const BlubBody &placement, const float *positions, uint32_t num_vertices, const uint32_t *indices,
                            uint32_t num_indices, float scale, BlubBody &stored) {
    MeshBodyHost m;
    m.props = mesh_body_properties(positions, num_vertices, indices, num_indices, scale, &m.vertices);
    m.indices.assign(indices, indices + num_indices);
    const BlubMeshBodyProperties &pr = m.props;
    // the placement's checks but the shape's (done above): finite values, density, quaternion norm
    BlubBody b = placement;
    b.shape = 0;
    for (int k = 0; k < 3; ++k) b.half_extent[k] = 1.0f;
    b = make_body_set(nullptr, &b, 1, false)[0]; // normalises the quaternion; dim == nullptr: the bounding box is checked below
    double qm[4] = {b.rotation[0], b.rotation[1], b.rotation[2], b.rotation[3]}, Rm[9];
    quat_rotation_f64(qm, Rm);
    const double *qp = pr.principal_rotation;
    const double q[4] = {qm[0] * qp[0] - qm[1] * qp[1] - qm[2] * qp[2] - qm[3] * qp[3], qm[0] * qp[1] + qm[1] * qp[0] + qm[2] * qp[3] - qm[3] * qp[2],
                         qm[0] * qp[2] - qm[1] * qp[3] + qm[2] * qp[0] + qm[3] * qp[1], qm[0] * qp[3] + qm[1] * qp[2] - qm[2] * qp[1] + qm[3] * qp[0]};
    const double qn = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    stored = b;
    stored.shape = 2;
    const bool model_frame = qp[0] == 1.0 && qp[1] == 0.0 && qp[2] == 0.0 && qp[3] == 0.0;
    for (int k = 0; k < 4 && !model_frame; ++k) stored.rotation[k] = (float)(q[k] / qn); // else the placement's, as set_bodies stores it
    for (int k = 0; k < 3; ++k) { // the centre of mass in the grid: c + R_model (scale * centroid)
        const double off = Rm[3 * k] * pr.centroid[0] + Rm[3 * k + 1] * pr.centroid[1] + Rm[3 * k + 2] * pr.centroid[2];
        stored.centre[k] = (float)((double)b.centre[k] + (double)scale * off);
        stored.half_extent[k] = 0.5f * (pr.bounds_hi[k] - pr.bounds_lo[k]);
    }
    m.props.mass = (float)((double)b.relative_density * pr.volume);
    for (int k = 0; k < 3; ++k) m.props.moments[k] = (float)((double)b.relative_density * pr.principal_moments[k]);
    if (!(m.props.mass > 0.0f) || !std::isfinite(m.props.mass)) refuse("the mass is not a positive float32");
    for (int k = 0; k < 3; ++k) {
        m.mid[k] = 0.5f * (pr.bounds_lo[k] + pr.bounds_hi[k]);
        if (!(m.props.moments[k] > 0.0f) || !std::isfinite(m.props.moments[k])) refuse("a principal moment is not a positive float32");
    }
    float e[3], off[3];
    mesh_body_box(stored, m.mid, e, off);
    if (dim)
        for (int k = 0; k < 3; ++k)
            if (stored.centre[k] + off[k] - e[k] < 1.0f || stored.centre[k] + off[k] + e[k] > (float)dim[k] - 1.0f)
                throw std::invalid_argument("set_bodies: a body's bounding box leaves [1, dim - 1]");
    return m;
}

void mesh_body_box(const BlubBody &b, const float mid[3], float e[3], float off[3]) {
    body_bounding_extents(b, e); // shape 2 takes the box branch: sum_j |R_kj| h_j
    const double q[4] = {b.rotation[0], b.rotation[1], b.rotation[2], b.rotation[3]};
    double R[9];
    quat_rotation_f64(q, R);
    for (int k = 0; k < 3; ++k) off[k] = (float)(R[3 * k] * mid[0] + R[3 * k + 1] * mid[1] + R[3 * k + 2] * mid[2]);
}

uint32_t mesh_body_cube_side(const float h[3], const float mid[3]) {
    double r = 0.0; // the farthest corner of the body-frame bounds from the centre of mass
    for (int c = 0; c < 8; ++c) {
        double s = 0.0;
        for (int k = 0; k < 3; ++k) {
            const double x = (double)mid[k] + ((c >> k & 1) ? (double)h[k] : -(double)h[k]);
            s += x * x;
        }
        r = std::max(r, std::sqrt(s));
    }
    return (uint32_t)std::ceil(2.0 * r) + 2u;
}

} // namespace blub
