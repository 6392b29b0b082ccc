// blub_run -- headless scene runner over the C ABI (include/blub_fluid.h only; links libblubcore.so).
//
// The reference has no headless mode; its closest thing to a batch run is the GUI's "fast forward"
// (src/simulation_controller.rs:96-157): batches of 16 steps, a device.poll(Maintain::Wait) after each batch, wall time
// logged as "Fast forward of {:?} took {:?} to compute".  This tool reproduces that protocol on an unchanged blub scene
// file, and stands in for three more pieces of the reference's shell (SURVEY.md section 8 f2-f4):
//   --stats FILE   solver statistics history as JSON (the GUI's residual / iteration plots, src/gui/mod.rs:177-210)
//   --trace FILE   one step as a Chrome trace with the reference's profiler scope labels (src/gui/mod.rs:487-491,
//                  hybrid_fluid.rs:780-973)
//   --dump FILE    particle positions (float32 x,y,z,pad) for an external viewer -- the renderer hand-off; pad holds the particle's tag bits
//                  (read it as uint32)
//                  (hybrid_fluid.rs:351-369) without wgpu
//   --record FPS PREFIX   the controller's "recording with fixed frame length" (simulation_controller.rs:80-82,174-176): the render
//                  clock advances by 1 / FPS per frame, the simulation runs the steps that belong to the frame (Timer::simulation_frame_loop),
//                  and instead of a screenshot the particle positions are written to PREFIX00000.f32, PREFIX00001.f32, ...
//   --save-state FILE  the fluid's complete state after the last step (blub_fluid_save_state); --checkpoint-every N also rewrites FILE every
//                  N steps at batch boundaries.  --load-state FILE resumes such a file instead of seeding the scene's fluid cubes: the scene
//                  still provides scale, origin and static objects, and the simulation clock restarts at step_count * dt.
//   --loads FILE   the history of the scene's solid load probes (fluid.load_probes) as JSON: the probes in grid cells and one record per
//                  step and probe, force in cells^4/s^2 and torque in cells^5/s^2 per unit density.  The device ring holds the newest 1024
//                  steps; the runner reads it at every batch or frame boundary, so a long run loses nothing.  With --load-state the scene's
//                  probes are set again (a state file holds none).
//   --bodies FILE  the trajectory of every floating body (fluid.bodies, or the bodies of a --load-state file) as JSON: one record per step
//                  and body with its load (as --loads) and its pose after the step, read from the device ring at every batch or frame boundary.
//   --models DIR   where the scene's static_objects find their OBJ files (the reference reads `models/<model>`,
//                  src/scene/models.rs:253).  Every step then runs Scene::step's order (src/scene/mod.rs:192-211): animate the
//                  models at the already advanced simulation time, voxelize their hulls, step the fluid.
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/blub_fluid.h"

static const char *kScopeLabels[14] = {
    "transfer particle velocity to grid", "compute divergence", "primary pressure solver (divergence)", "Particle Binning",
    "make velocity grid divergence free", "extrapolate velocity grid", "clear marker & linked list grids",
    "advect particles & write new linked list grid", "density projection: set boundary marker",
    "density projection: compute density error via gather", "secondary pressure solver (density)", "compute position change",
    "extrapolate velocity grid", "correct particle density error"};

static void die(const char *what) {
    std::fprintf(stderr, "blub_run: %s: %s\n", what, blub_last_error());
    std::exit(1);
}

int main(int argc, char **argv) {
    if (argc < 2) {
        std::fprintf(stderr, "usage: blub_run scene.json [--steps N] [--batch 16] [--hz 120] [--device 0] [--no-graph]\n"
                             "                [--stats out.json] [--trace out.json] [--dump particles.f32] [--models DIR] [--record FPS PREFIX]\n"
                             "                [--solver TOLERANCE MAX_ITERATIONS CHECK_FREQUENCY] [--rebin EVERY_N_STEPS]\n"
                             "                [--save-state FILE [--checkpoint-every N]] [--load-state FILE] [--loads out.json]\n"
                             "                [--bodies out.json]\n");
        return 2;
    }
    const char *scene = argv[1];
    int steps = 160, batch = 16, device = 0, graph = 1;
    long hz = 120;
    std::string bodies_path, loads_path, stats_path, trace_path, dump_path, models_dir = "models", record_prefix, save_path, load_path;
    double record_fps = 0.0;
    float solver_tol = -1.0f;
    int solver_max = 0, solver_freq = 0, rebin = -1, checkpoint_every = 0;
    for (int i = 2; i < argc; ++i) {
        auto next = [&](const char *flag) -> const char * {
            if (i + 1 >= argc) { std::fprintf(stderr, "blub_run: %s needs a value\n", flag); std::exit(2); }
            return argv[++i];
        };
        if (!std::strcmp(argv[i], "--steps")) steps = std::atoi(next("--steps"));
        else if (!std::strcmp(argv[i], "--batch")) batch = std::atoi(next("--batch"));
        else if (!std::strcmp(argv[i], "--hz")) hz = std::atol(next("--hz"));
        else if (!std::strcmp(argv[i], "--device")) device = std::atoi(next("--device"));
        else if (!std::strcmp(argv[i], "--no-graph")) graph = 0;
        else if (!std::strcmp(argv[i], "--stats")) stats_path = next("--stats");
        else if (!std::strcmp(argv[i], "--loads")) loads_path = next("--loads");
        else if (!std::strcmp(argv[i], "--bodies")) bodies_path = next("--bodies");
        else if (!std::strcmp(argv[i], "--trace")) trace_path = next("--trace");
        else if (!std::strcmp(argv[i], "--dump")) dump_path = next("--dump");
        else if (!std::strcmp(argv[i], "--models")) models_dir = next("--models");
        else if (!std::strcmp(argv[i], "--solver")) { solver_tol = (float)std::atof(next("--solver")); solver_max = std::atoi(next("--solver")); solver_freq = std::atoi(next("--solver")); }
        else if (!std::strcmp(argv[i], "--rebin")) rebin = std::atoi(next("--rebin"));
        else if (!std::strcmp(argv[i], "--save-state")) save_path = next("--save-state");
        else if (!std::strcmp(argv[i], "--checkpoint-every")) checkpoint_every = std::atoi(next("--checkpoint-every"));
        else if (!std::strcmp(argv[i], "--load-state")) load_path = next("--load-state");
        else if (!std::strcmp(argv[i], "--record")) { record_fps = std::atof(next("--record")); record_prefix = next("--record"); }
        else { std::fprintf(stderr, "blub_run: unknown option %s\n", argv[i]); return 2; }
    }
    if (steps < 1 || batch < 1 || hz < 1) { std::fprintf(stderr, "blub_run: bad --steps/--batch/--hz\n"); return 2; }
    // delta_from_steps_per_second: Duration::from_nanos(1e9 / hz), then as_secs_f32 (simulation_controller.rs:33-35)
    const uint64_t dt_ns = blub_simulation_delta_ns((uint64_t)hz);
    const double dt = (double)blub_duration_as_secs_f32(dt_ns);
    if (!record_prefix.empty() && !(record_fps > 0.0)) { std::fprintf(stderr, "blub_run: bad --record FPS\n"); return 2; }
    if (!record_prefix.empty() && !load_path.empty()) { std::fprintf(stderr, "blub_run: --load-state cannot resume a --record run\n"); return 2; }
    if (!loads_path.empty() && batch > BLUB_LOAD_HISTORY_LENGTH) {
        std::fprintf(stderr, "blub_run: --loads reads the load history at batch boundaries: --batch must not exceed %d\n", BLUB_LOAD_HISTORY_LENGTH);
        return 2;
    }
    if (!bodies_path.empty() && batch > BLUB_BODY_HISTORY_LENGTH) {
        std::fprintf(stderr, "blub_run: --bodies reads the body history at batch boundaries: --batch must not exceed %d\n", BLUB_BODY_HISTORY_LENGTH);
        return 2;
    }
    if (checkpoint_every < 0 || (checkpoint_every > 0 && save_path.empty())) {
        std::fprintf(stderr, "blub_run: --checkpoint-every needs a positive N and --save-state FILE\n");
        return 2;
    }

    BlubSceneInfo info;
    if (blub_scene_info(scene, &info)) die("cannot read scene");
    BlubFluid *fluid = nullptr;
    if (load_path.empty()) {
        if (blub_scene_load(&fluid, scene, device, nullptr)) die("cannot create fluid");
        blub_fluid_set_graph_replay(fluid, graph);
    } else { // the file holds every setting of the saved run; only options given on this command line override them
        BlubStateInfo state;
        if (blub_state_info(load_path.c_str(), &state)) die("cannot read the state file");
        if (std::memcmp(state.grid_dimension, info.grid_dimension, sizeof(state.grid_dimension)) != 0) {
            std::fprintf(stderr, "blub_run: the state file's grid %ux%ux%u is not the scene's %ux%ux%u\n", state.grid_dimension[0], state.grid_dimension[1],
                         state.grid_dimension[2], info.grid_dimension[0], info.grid_dimension[1], info.grid_dimension[2]);
            return 1;
        }
        if (blub_fluid_load_state(&fluid, load_path.c_str(), device, nullptr)) die("cannot load the state file");
        if (!graph) blub_fluid_set_graph_replay(fluid, 0);
        std::printf("resumed %s after step %u\n", load_path.c_str(), blub_fluid_step_count(fluid));
    }
    if (solver_max > 0) { // the GUI's solver sliders (src/gui/mod.rs:228-250) write the same two SolverConfig structs
        for (int which = 0; which < 2; ++which) {
            BlubSolverConfig *c = blub_fluid_solver_config(fluid, which);
            c->error_tolerance = solver_tol;
            c->max_num_iterations = solver_max;
            c->error_check_frequency = solver_freq > 0 ? solver_freq : 4;
        }
    }
    if (rebin >= 0) *blub_fluid_rebinning_frequency(fluid) = (uint32_t)rebin;
    BlubLoadProbe probes[BLUB_LOAD_PROBES_MAX];
    uint32_t num_probes = 0;
    if (blub_scene_load_probes(scene, probes, BLUB_LOAD_PROBES_MAX, &num_probes)) die("cannot read the scene's load probes");
    if (!load_path.empty() && num_probes && blub_fluid_set_load_probes(fluid, probes, num_probes)) die("cannot set the load probes");
    std::printf("scene %s: grid %ux%ux%u, %u particles (max %u), %u static object(s), dt %.9f s\n", scene, info.grid_dimension[0],
                info.grid_dimension[1], info.grid_dimension[2], blub_fluid_num_particles(fluid), info.max_num_particles, info.num_static_objects, dt);

    // SceneModels::from_config (src/scene/models.rs:240-262): one mesh per static object
    struct Solid { BlubMesh *mesh; BlubRigidObject placement; };
    std::vector<Solid> solids;
    void *voxels = nullptr;
    for (uint32_t k = 0; k < info.num_static_objects; ++k) {
        Solid s;
        char model[1024];
        if (blub_scene_static_object(scene, k, &s.placement, model, sizeof(model))) die("cannot read static object");
        const std::string path = models_dir + "/" + model;
        if (blub_mesh_load_obj(&s.mesh, path.c_str(), device)) die("cannot load model"); // the reference fails to load the scene as well
        uint32_t nv = 0, nt = 0;
        blub_mesh_info(s.mesh, &nv, &nt);
        std::printf("static object %u: %s, %u vertices, %u triangles\n", k, path.c_str(), nv, nt);
        solids.push_back(s);
    }
    if (!solids.empty()) {
        const size_t cells = (size_t)info.grid_dimension[0] * info.grid_dimension[1] * info.grid_dimension[2];
        if (blub_device_malloc(&voxels, cells * 8, device)) die("cannot allocate the voxel volume");
        if (blub_fluid_set_solid_voxels(fluid, voxels)) die("set_solid_voxels failed");
    }
    // Timer::total_simulated_time / total_rendered_time; a resumed run continues the clock, so that animated solids are where they were
    uint64_t simulated_ns = (uint64_t)blub_fluid_step_count(fluid) * dt_ns, rendered_ns = 0;
    auto scene_step = [&]() {
        simulated_ns += dt_ns; // advanced BEFORE the step it belongs to (src/timer.rs:122-124)
        const double simulated = (double)blub_duration_as_secs_f32(simulated_ns);
        for (size_t k = 0; k < solids.size(); ++k)
            if (blub_solid_voxelize_mesh(voxels, info.grid_dimension, solids[k].mesh, &solids[k].placement, info.grid_to_world_scale, info.world_position,
                                         simulated, dt, k == 0, blub_fluid_stream(fluid), nullptr))
                die("voxelization failed");
        if (blub_fluid_step(fluid, dt)) die("step failed");
    };

    auto write_particles = [&](const std::string &path) {
        const uint32_t n = blub_fluid_num_particles(fluid);
        std::vector<float> pos((size_t)n * 4);
        if (n && blub_fluid_download(fluid, BLUB_TAP_PARTICLE_POS, pos.data(), pos.size() * sizeof(float))) die("download failed");
        FILE *f = std::fopen(path.c_str(), "wb");
        if (!f) { std::perror("blub_run: cannot write particles"); std::exit(1); }
        std::fwrite(pos.data(), sizeof(float), pos.size(), f);
        std::fclose(f);
        return n;
    };

    // every record of every probe, collected at batch / frame boundaries (the ring holds the newest BLUB_LOAD_HISTORY_LENGTH steps)
    std::vector<std::vector<BlubSolidLoad>> loads(num_probes);
    std::vector<BlubSolidLoad> ring(BLUB_LOAD_HISTORY_LENGTH);
    auto collect_loads = [&]() {
        if (loads_path.empty()) return;
        for (uint32_t p = 0; p < num_probes; ++p) {
            uint32_t n = 0;
            if (blub_fluid_load_history(fluid, p, ring.data(), BLUB_LOAD_HISTORY_LENGTH, &n)) die("cannot read the load history");
            for (uint32_t k = 0; k < n; ++k)
                if (loads[p].empty() || ring[k].step > loads[p].back().step) loads[p].push_back(ring[k]);
        }
    };

    // every record of every body, collected the same way (a state file's bodies are the fluid's own: nothing to set again)
    BlubBody bodies[BLUB_BODIES_MAX];
    uint32_t num_bodies = 0;
    if (blub_fluid_bodies(fluid, bodies, BLUB_BODIES_MAX, &num_bodies)) die("cannot read the bodies");
    std::vector<std::vector<BlubBodyRecord>> trajectories(num_bodies);
    std::vector<BlubBodyRecord> body_ring(BLUB_BODY_HISTORY_LENGTH);
    auto collect_bodies = [&]() {
        if (bodies_path.empty()) return;
        for (uint32_t b = 0; b < num_bodies; ++b) {
            uint32_t n = 0;
            if (blub_fluid_body_history(fluid, b, body_ring.data(), BLUB_BODY_HISTORY_LENGTH, &n)) die("cannot read the body history");
            for (uint32_t k = 0; k < n; ++k)
                if (trajectories[b].empty() || body_ring[k].step > trajectories[b].back().step) trajectories[b].push_back(body_ring[k]);
        }
    };

    const bool has_flow = blub_fluid_has_flow(fluid) == 1;
    int done = 0, saved_at = -1;
    auto save_state = [&]() {
        if (blub_fluid_save_state(fluid, save_path.c_str())) die("cannot save the state");
        saved_at = done;
        std::printf("saved the state after step %u to %s\n", blub_fluid_step_count(fluid), save_path.c_str());
    };
    auto checkpoint = [&]() { // at batch / frame boundaries only
        if (checkpoint_every > 0 && done - (saved_at < 0 ? 0 : saved_at) >= checkpoint_every) save_state();
    };

    const auto t0 = std::chrono::steady_clock::now();
    if (!record_prefix.empty()) { // RecordingWithFixedFrameLength: one frame = 1 / FPS on the render clock
        const uint64_t frame_ns = (uint64_t)(1e9 / record_fps); // Duration::from_secs_f64(1.0 / fps), truncated to nanoseconds
        uint64_t clock_ns = 0; // the Timer's own simulation clock; scene_step keeps the same count in simulated_ns
        for (int frame = 0; done < steps; ++frame) {
            uint32_t n = blub_timer_steps_in_frame(&rendered_ns, &clock_ns, frame_ns, dt_ns);
            if ((int)n > steps - done) n = (uint32_t)(steps - done);
            for (uint32_t k = 0; k < n; ++k) scene_step();
            if (blub_fluid_synchronize(fluid)) die("synchronize failed");
            blub_fluid_update_statistics(fluid);
            done += (int)n;
            char name[32];
            std::snprintf(name, sizeof(name), "%05d.f32", frame);
            write_particles(record_prefix + name);
            collect_loads();
            collect_bodies();
            std::printf("frame %d: %u step(s), simulated %.6f s\n", frame, n, (double)blub_duration_as_secs_f32(simulated_ns));
            checkpoint();
        }
    }
    while (done < steps) { // MAX_FAST_FORWARD_SIMULATION_BATCH_SIZE = 16, then wait for the GPU
        const int n = steps - done < batch ? steps - done : batch;
        for (int k = 0; k < n; ++k) scene_step();
        if (blub_fluid_synchronize(fluid)) die("synchronize failed");
        blub_fluid_update_statistics(fluid);
        done += n;
        collect_loads();
        collect_bodies();
        if (has_flow) // sources and drains change the particle count as the run goes
            std::printf("simulation fast forwarding batch finished (progress %d/%d, %u particles)\n", done, steps, blub_fluid_num_particles(fluid));
        else
            std::printf("simulation fast forwarding batch finished (progress %d/%d)\n", done, steps);
        checkpoint();
    }
    const double secs = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    std::printf("Fast forward of %.6fs took %.6fs to compute (%.2f steps/s)\n", steps * dt, secs, steps / secs);

    if (!save_path.empty() && saved_at != done) save_state(); // before the extra timed step of --trace

    if (!stats_path.empty()) {
        FILE *f = std::fopen(stats_path.c_str(), "w");
        if (!f) { std::perror("blub_run: --stats"); return 1; }
        std::fprintf(f, "{\"steps\": %d, \"seconds\": %.6f", steps, secs);
        const char *names[2] = {"velocity", "density"};
        for (int which = 0; which < 2; ++which) {
            BlubSolverSample s[100];
            const size_t n = blub_fluid_solver_stats(fluid, which, s, 100);
            std::fprintf(f, ", \"%s\": [", names[which]);
            for (size_t k = 0; k < n; ++k) std::fprintf(f, "%s{\"error\": %.9g, \"iteration_count\": %d}", k ? ", " : "", s[k].error, s[k].iteration_count);
            std::fprintf(f, "]");
        }
        if (has_flow) {
            uint64_t c[3] = {0, 0, 0};
            if (blub_fluid_flow_counters(fluid, c)) die("cannot read the flow counters");
            std::fprintf(f, ", \"flow\": {\"emitted\": %llu, \"drained\": %llu, \"refused\": %llu}", (unsigned long long)c[0], (unsigned long long)c[1],
                         (unsigned long long)c[2]);
        }
        BlubViscosity visc;
        if (blub_fluid_viscosity(fluid, &visc)) die("cannot read the viscosity");
        if (visc.kinematic_viscosity > 0.0f) {
            int32_t it = 0;
            float e[3] = {0, 0, 0};
            if (blub_fluid_last_viscosity_solve(fluid, &it, e)) die("cannot read the last viscosity solve");
            std::fprintf(f, ", \"viscosity\": {\"kinematic_viscosity\": %.9g, \"last_iterations\": %d, \"last_max_error\": [%.9g, %.9g, %.9g]}",
                         visc.kinematic_viscosity, it, e[0], e[1], e[2]);
        }
        std::fprintf(f, "}\n");
        std::fclose(f);
    }
    if (!loads_path.empty()) {
        FILE *f = std::fopen(loads_path.c_str(), "w");
        if (!f) { std::perror("blub_run: --loads"); return 1; }
        const double fs = (double)(1 << BLUB_LOAD_FORCE_FRAC_BITS), ts = (double)(1 << BLUB_LOAD_TORQUE_FRAC_BITS);
        std::fprintf(f, "{\"grid_to_world_scale\": %.9g, \"dt\": %.9g, \"force_units\": \"cells^4/s^2 per unit density\", "
                        "\"torque_units\": \"cells^5/s^2 per unit density\", \"probes\": [",
                     info.grid_to_world_scale, dt);
        for (uint32_t p = 0; p < num_probes; ++p) {
            const BlubLoadProbe &q = probes[p];
            std::fprintf(f, "%s\n {\"min\": [%.9g, %.9g, %.9g], \"max\": [%.9g, %.9g, %.9g], \"pivot\": [%.9g, %.9g, %.9g], \"records\": [", p ? "," : "",
                         q.min_grid[0], q.min_grid[1], q.min_grid[2], q.max_grid[0], q.max_grid[1], q.max_grid[2], q.pivot_grid[0], q.pivot_grid[1], q.pivot_grid[2]);
            for (size_t k = 0; k < loads[p].size(); ++k) {
                const BlubSolidLoad &r = loads[p][k];
                std::fprintf(f, "%s\n  {\"step\": %u, \"wetted_faces\": %u, \"force\": [%.17g, %.17g, %.17g], \"torque\": [%.17g, %.17g, %.17g]}", k ? "," : "",
                             r.step, r.wetted_faces, r.force_fx[0] / fs, r.force_fx[1] / fs, r.force_fx[2] / fs, r.torque_fx[0] / ts, r.torque_fx[1] / ts,
                             r.torque_fx[2] / ts);
            }
            std::fprintf(f, "]}");
        }
        std::fprintf(f, "\n]}\n");
        std::fclose(f);
    }
    if (!bodies_path.empty()) {
        FILE *f = std::fopen(bodies_path.c_str(), "w");
        if (!f) { std::perror("blub_run: --bodies"); return 1; }
        const double fs = (double)(1 << BLUB_LOAD_FORCE_FRAC_BITS), ts = (double)(1 << BLUB_LOAD_TORQUE_FRAC_BITS);
        std::fprintf(f, "{\"grid_to_world_scale\": %.9g, \"dt\": %.9g, \"units\": \"cells, cells/s, rad/s; force cells^4/s^2 and torque cells^5/s^2 per unit density\", "
                        "\"bodies\": [",
                     info.grid_to_world_scale, dt);
        for (uint32_t b = 0; b < num_bodies; ++b) {
            const BlubBody &o = bodies[b];
            std::fprintf(f, "%s\n {\"shape\": \"%s\", \"half_extent\": [%.9g, %.9g, %.9g], \"relative_density\": %.9g, \"records\": [", b ? "," : "",
                         o.shape == 1 ? "sphere" : "box", o.half_extent[0], o.half_extent[1], o.half_extent[2], o.relative_density);
            for (size_t k = 0; k < trajectories[b].size(); ++k) {
                const BlubBodyRecord &r = trajectories[b][k];
                std::fprintf(f,
                             "%s\n  {\"step\": %u, \"wetted_faces\": %u, \"force\": [%.17g, %.17g, %.17g], \"torque\": [%.17g, %.17g, %.17g], "
                             "\"centre\": [%.9g, %.9g, %.9g], \"rotation\": [%.9g, %.9g, %.9g, %.9g], \"velocity\": [%.9g, %.9g, %.9g], "
                             "\"angular_velocity\": [%.9g, %.9g, %.9g]}",
                             k ? "," : "", r.step, r.wetted_faces, r.force_fx[0] / fs, r.force_fx[1] / fs, r.force_fx[2] / fs, r.torque_fx[0] / ts,
                             r.torque_fx[1] / ts, r.torque_fx[2] / ts, r.centre[0], r.centre[1], r.centre[2], r.rotation[0], r.rotation[1], r.rotation[2],
                             r.rotation[3], r.velocity[0], r.velocity[1], r.velocity[2], r.angular_velocity[0], r.angular_velocity[1], r.angular_velocity[2]);
            }
            std::fprintf(f, "]}");
        }
        std::fprintf(f, "\n]}\n");
        std::fclose(f);
    }
    if (!trace_path.empty()) { // "Write Chrometrace" (src/gui/mod.rs:487-491): one eagerly launched, event-timed step
        float ms[14];
        if (blub_fluid_step_timed(fluid, dt, ms)) die("timed step failed");
        FILE *f = std::fopen(trace_path.c_str(), "w");
        if (!f) { std::perror("blub_run: --trace"); return 1; }
        std::fprintf(f, "{\"traceEvents\": [\n");
        double ts = 0.0, total = 0.0;
        for (int s = 0; s < 14; ++s) total += ms[s];
        std::fprintf(f, " {\"name\": \"HybridFluid step\", \"ph\": \"X\", \"pid\": 1, \"tid\": 1, \"ts\": 0, \"dur\": %.3f}", total * 1e3);
        for (int s = 0; s < 14; ++s) {
            std::fprintf(f, ",\n {\"name\": \"%s\", \"ph\": \"X\", \"pid\": 1, \"tid\": 1, \"ts\": %.3f, \"dur\": %.3f}", kScopeLabels[s], ts, ms[s] * 1e3);
            ts += ms[s] * 1e3;
        }
        std::fprintf(f, "\n]}\n");
        std::fclose(f);
    }
    if (!dump_path.empty()) {
        const uint32_t n = write_particles(dump_path);
        std::printf("wrote %u particles (float32 x y z pad, grid units; world = grid * %g + (%g, %g, %g)) to %s\n", n, info.grid_to_world_scale,
                    info.world_position[0], info.world_position[1], info.world_position[2], dump_path.c_str());
    }
    blub_fluid_destroy(fluid);
    for (Solid &s : solids) blub_mesh_destroy(s.mesh);
    if (voxels) blub_device_free(voxels);
    return 0;
}
