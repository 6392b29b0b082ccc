// mesh_voxelizer.cu -- conservative HULL voxelization of triangle meshes into the RGBA16F solid-voxel volume (SURVEY.md section 8 f1).
//
// Replaces the reference's voxelization render pass (src/scene/voxelization.rs:118-157: clear, then one draw per mesh with hardware
// conservative rasterization along each triangle's dominant axis; shader/voxelize/conservative_hull.{vert,frag}).  There is no raster
// pipeline on this path: one thread block per triangle walks the triangle's pixel range and evaluates, per pixel, exactly what the
// fragment shader evaluates (voxelize_core.hpp, shared with the host twin the CPU tests use).  Two passes make the result
// deterministic where the reference's unordered image stores are not: pass 1 takes, per voxel, the maximum of
// (triangle, store kind, pixel) over all stores that hit it (64-bit atomicMax); pass 2 lets exactly that store write the voxel --
// the outcome of executing the draw sequentially.  Compiled with -fmad=false so that host twin, NumPy restatement and device agree
// bit for bit on every floor() / comparison.
#include <cmath>
#include <cstring>
#include <fstream>
#include <sstream>
#include <string>
#include <vector>

#include "../../include/blub_fluid.h"
#include "blub_core.hpp"
#include "voxelize_core.hpp"

struct BlubMesh {
    int device = 0;
    uint32_t num_vertices = 0, num_triangles = 0;
    float *positions = nullptr;     // device, xyz per vertex (model space)
    uint32_t *indices = nullptr;    // device, 3 per triangle
    unsigned long long *owner = nullptr; // device scratch, one word per voxel of the last grid size used
    size_t owner_cells = 0;
};

namespace blub {
namespace {

constexpr int VOX_THREADS = 64;

template <bool RESOLVE>
__global__ void __launch_bounds__(VOX_THREADS) voxelize_mesh_kernel(const float *__restrict__ positions, const uint32_t *__restrict__ indices,
                                                                    uint32_t num_triangles, vox::MeshPose pose, int nx, int ny, int nz, int viewport,
                                                                    unsigned long long *__restrict__ owner, uint2 *__restrict__ voxels) {
    const int res[3] = {nx, ny, nz};
    for (uint32_t t = blockIdx.x; t < num_triangles; t += gridDim.x) {
        float v[3][3];
#pragma unroll
        for (int k = 0; k < 3; ++k) vox::transform_vertex(pose, positions + 3 * (size_t)indices[3 * (size_t)t + k], v[k]);
        vox::TriSetup s;
        if (!vox::setup_triangle(v[0], v[1], v[2], viewport, s)) continue;
        const int w = s.x1 - s.x0 + 1, h = s.y1 - s.y0 + 1;
        if (w <= 0 || h <= 0) continue;
        for (int idx = threadIdx.x; idx < w * h; idx += VOX_THREADS) {
            const int px = s.x0 + idx % w, py = s.y0 + idx / w;
            if (!vox::pixel_overlaps(s, px, py)) continue;
            vox::Fragment f;
            vox::shade_fragment(s, pose, res, viewport, px, py, f);
            for (int k = 0; k < f.count; ++k) {
                const size_t cell = ((size_t)f.cell[k][2] * ny + f.cell[k][1]) * nx + f.cell[k][0];
                const unsigned long long prio = ((unsigned long long)(4ull * t + (unsigned)f.kind[k] + 1ull) << 32) | (unsigned)(py * viewport + px);
                if (!RESOLVE) {
                    atomicMax(owner + cell, prio);
                } else if (owner[cell] == prio) {
                    __half2 lo = __floats2half2_rn(f.vel[k][0], f.vel[k][1]), hi = __floats2half2_rn(f.vel[k][2], 1.0f);
                    voxels[cell] = make_uint2(*reinterpret_cast<unsigned *>(&lo), *reinterpret_cast<unsigned *>(&hi));
                }
            }
        }
    }
}

// StaticMeshData::to_gpu, src/scene/models.rs:186-224, from the animation state solids.cu evaluates
vox::MeshPose pose_from_state(const BlubRigidObject &o, const BlubRigidState &st, float grid_to_world_scale) {
    vox::MeshPose p;
    const float k = o.scale / grid_to_world_scale; // Scale(1 / grid_to_world_scale) * Translate * Translate * Scale(scale) * Rotation
    for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) p.m[4 * r + c] = st.rotation[3 * r + c] * k;
        p.m[4 * r + 3] = st.centre_voxel[r];
        p.centre[r] = st.centre_voxel[r];
        p.axis[r] = st.axis_scaled[r];
        p.velocity[r] = st.velocity_voxel[r];
    }
    return p;
}

} // namespace

void rigid_state_at(const BlubRigidObject &o, float grid_to_world_scale, const float fluid_world_position[3], double total_time, double delta,
                    BlubRigidState &out); // solids.cu

void voxelize_mesh(void *rgba16f, const uint32_t dim[3], BlubMesh &mesh, const BlubRigidObject &o, float grid_to_world_scale, const float fluid_world_position[3],
                   double total_time, double delta, int clear_first, cudaStream_t stream, BlubRigidState *state_out) {
    BLUB_CUDA_CHECK(cudaSetDevice(mesh.device)); // the volume and the stream must live on the mesh's device
    BlubRigidState st;
    rigid_state_at(o, grid_to_world_scale, fluid_world_position, total_time, delta, st);
    if (state_out) *state_out = st;
    const vox::MeshPose pose = pose_from_state(o, st, grid_to_world_scale);
    const size_t cells = (size_t)dim[0] * dim[1] * dim[2];
    if (mesh.owner_cells < cells) {
        if (mesh.owner) BLUB_CUDA_CHECK(cudaFree(mesh.owner));
        mesh.owner = nullptr;
        mesh.owner_cells = 0;
        BLUB_CUDA_CHECK(cudaMalloc(&mesh.owner, cells * sizeof(unsigned long long)));
        mesh.owner_cells = cells;
    }
    if (clear_first) BLUB_CUDA_CHECK(cudaMemsetAsync(rgba16f, 0, cells * 8, stream)); // encoder.clear_texture, voxelization.rs:125
    if (mesh.num_triangles == 0) return;
    BLUB_CUDA_CHECK(cudaMemsetAsync(mesh.owner, 0, cells * sizeof(unsigned long long), stream));
    const int viewport = (int)std::max(dim[0], std::max(dim[1], dim[2])); // voxelization.rs:100
    const int blocks = (int)std::min<uint32_t>(mesh.num_triangles, 1u << 20);
    BLUB_LAUNCH(voxelize_mesh_kernel<false>, blocks, VOX_THREADS, 0, stream, mesh.positions, mesh.indices, mesh.num_triangles, pose, (int)dim[0], (int)dim[1],
                (int)dim[2], viewport, mesh.owner, static_cast<uint2 *>(rgba16f));
    BLUB_LAUNCH(voxelize_mesh_kernel<true>, blocks, VOX_THREADS, 0, stream, mesh.positions, mesh.indices, mesh.num_triangles, pose, (int)dim[0], (int)dim[1],
                (int)dim[2], viewport, mesh.owner, static_cast<uint2 *>(rgba16f));
}

BlubMesh *mesh_create(const float *positions, uint32_t num_vertices, const uint32_t *indices, uint32_t num_indices, int device) {
    if (num_indices % 3 != 0) throw std::invalid_argument("mesh: the index count must be a multiple of 3");
    if ((num_vertices && !positions) || (num_indices && !indices)) throw std::invalid_argument("mesh: NULL vertex / index array");
    for (uint32_t k = 0; k < num_indices; ++k)
        if (indices[k] >= num_vertices) throw std::invalid_argument("mesh: index " + std::to_string(indices[k]) + " out of range");
    BLUB_CUDA_CHECK(cudaSetDevice(device));
    BlubMesh *m = new BlubMesh();
    m->device = device;
    m->num_vertices = num_vertices;
    m->num_triangles = num_indices / 3;
    try {
        BLUB_CUDA_CHECK(cudaMalloc(&m->positions, std::max<size_t>(1, (size_t)num_vertices * 12)));
        BLUB_CUDA_CHECK(cudaMalloc(&m->indices, std::max<size_t>(1, (size_t)num_indices * 4)));
        if (num_vertices) BLUB_CUDA_CHECK(cudaMemcpy(m->positions, positions, (size_t)num_vertices * 12, cudaMemcpyHostToDevice));
        if (num_indices) BLUB_CUDA_CHECK(cudaMemcpy(m->indices, indices, (size_t)num_indices * 4, cudaMemcpyHostToDevice));
    } catch (...) {
        mesh_destroy(m);
        throw;
    }
    return m;
}

void mesh_info(const BlubMesh &m, uint32_t &num_vertices, uint32_t &num_triangles) {
    num_vertices = m.num_vertices;
    num_triangles = m.num_triangles;
}

int mesh_device(const BlubMesh &m) { return m.device; }

void mesh_download(const BlubMesh &m, std::vector<float> &positions, std::vector<uint32_t> &indices) {
    positions.resize(3 * (size_t)m.num_vertices);
    indices.resize(3 * (size_t)m.num_triangles);
    BLUB_CUDA_CHECK(cudaSetDevice(m.device));
    if (m.num_vertices) BLUB_CUDA_CHECK(cudaMemcpy(positions.data(), m.positions, positions.size() * sizeof(float), cudaMemcpyDeviceToHost));
    if (m.num_triangles) BLUB_CUDA_CHECK(cudaMemcpy(indices.data(), m.indices, indices.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost));
}

void mesh_destroy(BlubMesh *m) {
    if (!m) return;
    if (m->positions) cudaFree(m->positions);
    if (m->indices) cudaFree(m->indices);
    if (m->owner) cudaFree(m->owner);
    delete m;
}

// Wavefront OBJ geometry as tobj::load_obj(triangulate, ignore_points, ignore_lines) delivers it to the reference
// (src/scene/models.rs:252-262): `v x y z` positions and `f` polygons fan-triangulated around their first corner; corners are
// v, v/vt, v//vn or v/vt/vn with 1-based or negative (relative) position indices.  Everything else (normals, uvs, groups, materials)
// does not reach the voxelizer and is skipped.
void read_obj(const std::string &path, std::vector<float> &positions, std::vector<uint32_t> &indices) {
    std::ifstream in(path);
    if (!in) throw std::runtime_error("cannot open OBJ file " + path);
    positions.clear();
    indices.clear();
    std::string line;
    size_t lineno = 0;
    while (std::getline(in, line)) {
        ++lineno;
        const size_t hash = line.find('#');
        if (hash != std::string::npos) line.resize(hash);
        std::istringstream ss(line);
        std::string tag;
        if (!(ss >> tag)) continue;
        if (tag == "v") {
            float x, y, z;
            if (!(ss >> x >> y >> z)) throw std::runtime_error(path + ":" + std::to_string(lineno) + ": malformed vertex");
            positions.push_back(x);
            positions.push_back(y);
            positions.push_back(z);
        } else if (tag == "f") {
            std::vector<uint32_t> corners;
            std::string corner;
            while (ss >> corner) {
                long idx = 0;
                try {
                    idx = std::stol(corner.substr(0, corner.find('/')));
                } catch (...) {
                    throw std::runtime_error(path + ":" + std::to_string(lineno) + ": malformed face corner `" + corner + "`");
                }
                const long count = (long)(positions.size() / 3);
                const long resolved = idx > 0 ? idx - 1 : count + idx;
                if (idx == 0 || resolved < 0 || resolved >= count)
                    throw std::runtime_error(path + ":" + std::to_string(lineno) + ": vertex index " + std::to_string(idx) + " out of range");
                corners.push_back((uint32_t)resolved);
            }
            if (corners.size() < 3) continue; // points and lines are ignored (LoadOptions::ignore_points / ignore_lines)
            for (size_t k = 1; k + 1 < corners.size(); ++k) {
                indices.push_back(corners[0]);
                indices.push_back(corners[k]);
                indices.push_back(corners[k + 1]);
            }
        }
    }
}

} // namespace blub
