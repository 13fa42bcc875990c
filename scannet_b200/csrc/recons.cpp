// `recons` — the reconstruction stage of the reference pipeline in library form:
//   FriedLiver.exe <params.txt> <params2.txt> <file.sens>          (Server/scan_processor.py:27-29,123-126)
// Every frame of the stream is decoded on the GPU (depth by the inflate kernel, colour by the device JPEG decoder registered to
// the depth image, as `fuse` does), tracked against the model and integrated at its tracked pose (csrc/track.cu, DESIGN.md §6j);
// then marching cubes -> <base>.ply and the trajectory -> the .sens (s_overwriteOrigSensTrajectory, zParametersScanNet.txt:5):
// only the 64-byte pose fields change, the payloads are written back byte for byte.  Nothing is written when a call fails.
// Not BundleFusion: no sparse features; the dense global optimisation of DESIGN.md §6k runs only with --global
// (scn_recons_scene_global).
#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "scn_common.h"

namespace {

using scn::now_s;
using TsdfPtr = std::unique_ptr<scn_tsdf, scn::Release<scn_tsdf_destroy>>;
using TrackPtr = std::unique_ptr<scn_track, scn::Release<scn_track_destroy>>;
using GlobalPtr = std::unique_ptr<scn_globalopt, scn::Release<scn_globalopt_destroy>>;

constexpr uint32_t kChunk = 256;                    // frames decoded per call of the depth and colour decoders

// T_f' = T_k' (T_k^-1 T_f): T_k^-1 = [R^T | -R^T t] and both products in binary64, rounded once
void propagate(const float* Tk, const float* Tk_new, const float* Tf, float* out) {
  double A[12];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 4; ++c) {
      double m = ((double)Tk[r] * Tf[c] + (double)Tk[4 + r] * Tf[4 + c]) + (double)Tk[8 + r] * Tf[8 + c];
      if (c == 3) m = m - (((double)Tk[r] * Tk[3] + (double)Tk[4 + r] * Tk[7]) + (double)Tk[8 + r] * Tk[11]);
      A[4 * r + c] = m;
    }
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 4; ++c) {
      double m = ((double)Tk_new[4 * r] * A[c] + (double)Tk_new[4 * r + 1] * A[4 + c]) + (double)Tk_new[4 * r + 2] * A[8 + c];
      if (c == 3) m = m + (double)Tk_new[4 * r + 3];
      out[4 * r + c] = (float)m;
    }
  out[12] = 0.f; out[13] = 0.f; out[14] = 0.f; out[15] = 1.f;
}

// gparams non-null: the keyframes go to the global optimiser as each chunk is tracked; after the last chunk the solve, the
// propagation to every tracked frame, and the re-integration of the stream at the new poses through fuse's scene driver
int recons_scene(const char* sens_path, const char* out_ply, const char* out_sens, const scn_tsdf_params* params,
                 const scn_track_params* tparams, const scn_globalopt_params* gparams, int device, scn_recons_report_t& rep,
                 scn_globalopt_report_t* grep) {
  const double t_begin = now_s();
  rep.device = device;
  if (int r = scn_set_device(device)) return r;
  scn_sens* sp = nullptr;
  if (int r = scn_sens_open(sens_path, &sp)) return r;
  scn::SensPtr sens(sp);
  scn_sens_info_t in; scn_sens_info(sp, &in);
  rep.frames = in.n_frames;
  if (in.depth_compression != 0 && in.depth_compression != 1)
    return scn::fail(SCN_ERR_UNSUPPORTED, "depth compression %d is not decoded on the GPU", in.depth_compression);
  scn_tsdf_params p = *params;
  p.width = in.depth_width; p.height = in.depth_height; p.depth_shift = in.depth_shift;
  p.batch_frames = 1;                               // one frame per integration: the next frame is tracked against it
  scn_tsdf* vp = nullptr;
  if (int r = scn_tsdf_create(&p, device, &vp)) return r;
  TsdfPtr vol(vp);
  scn_track* tp = nullptr;
  if (int r = scn_track_create(vp, tparams, &tp)) return r;
  TrackPtr tr(tp);
  GlobalPtr gopt;
  if (gparams) {
    scn_globalopt* gp = nullptr;
    if (int r = scn_globalopt_create(vp, gparams, &gp)) return r;
    gopt.reset(gp);
  }
  std::vector<uint64_t> kf_frame;                    // frame of each keyframe, in order
  std::vector<int64_t> kf_of_submap;                 // keyframe index of each submap, -1 while it has none
  const bool use_color = in.color_compression <= 2 && in.color_width > 0 && in.color_height > 0;
  const size_t px = (size_t)in.depth_width * in.depth_height;
  const uint32_t CH = (uint32_t)std::min<uint64_t>(kChunk, std::max<uint64_t>(in.n_frames, 1));
  scn::DevicePtr<uint16_t> d_depth((uint16_t*)scn_device_alloc((size_t)CH * px * 2));
  scn::DevicePtr<uint8_t> d_rgb(use_color ? (uint8_t*)scn_device_alloc((size_t)CH * px * 3) : nullptr);
  scn::DevicePtr<int32_t> d_lut(use_color ? (int32_t*)scn_device_alloc(px * 4) : nullptr);
  if (!d_depth || (use_color && (!d_rgb || !d_lut))) return scn::fail(SCN_ERR_CUDA, "device allocation of the frame buffers failed");
  if (use_color) {
    std::vector<int32_t> lut;
    scn::build_color_lut(in, lut);
    if (int r = scn_memcpy_h2d(d_lut.get(), lut.data(), px * 4, nullptr)) return r;
  }
  float first[16];
  if (in.n_frames) { if (int r = scn_sens_frame_meta(sp, 0, first, nullptr, nullptr, nullptr, nullptr)) return r; }
  std::vector<scn_track_frame_t> res(in.n_frames);
  std::vector<uint64_t> frames;
  rep.setup_s = now_s() - t_begin;
  const double t0 = now_s();
  for (uint64_t f0 = 0; f0 < in.n_frames; f0 += CH) {
    const uint32_t n = (uint32_t)std::min<uint64_t>(CH, in.n_frames - f0);
    double td = now_s();
    frames.resize(n);
    for (uint32_t i = 0; i < n; ++i) frames[i] = f0 + i;
    if (int r = scn::sens_depth_to_device(sp, frames.data(), n, d_depth.get(), nullptr)) return r;
    if (use_color) {
      uint32_t k = 0;
      if (int r = scn_sens_decode_color_device(sp, f0, n, d_lut.get(), (uint32_t)px, d_rgb.get(), nullptr, &k)) return r;
    }
    rep.decode_s += now_s() - td;
    td = now_s();
    if (int r = scn_track_frames(tp, n, d_depth.get(), d_rgb.get(), in.depth_intrinsic, first, res.data() + f0)) return r;
    rep.track_s += now_s() - td;
    if (gopt) {                                      // a submap's keyframe is its first tracked frame; submaps span chunks
      const uint64_t S = gparams->submap_size;
      for (uint32_t i = 0; i < n; ++i) {
        const uint64_t f = f0 + i, sm = f / S;
        if (kf_of_submap.size() <= sm) kf_of_submap.resize(sm + 1, -1);
        if (res[f].lost || kf_of_submap[sm] >= 0) continue;
        if (int r = scn_globalopt_add_keyframes(gopt.get(), 1, d_depth.get() + i * px, res[f].cam2world, in.depth_intrinsic)) return r;
        kf_of_submap[sm] = (int64_t)kf_frame.size();
        kf_frame.push_back(f);
      }
    }
  }
  rep.recons_s = now_s() - t0;
  for (const scn_track_frame_t& r : res) rep.frames_lost += r.lost;
  rep.frames_tracked = in.n_frames - rep.frames_lost;
  scn_track_phase_ms(tp, &rep.filter_pyramid_ms, &rep.icp_ms, &rep.integrate_ms, &rep.raycast_ms);
  scn_track_stats(tp, nullptr, &rep.kernel_launches);
  scn_tsdf_stats_t st; scn_tsdf_stats(vp, &st);
  rep.blocks_allocated = st.blocks_allocated;
  bool reintegrate = false;
  if (gopt) {
    std::vector<float> kp(kf_frame.size() * 16 + 16);
    scn_globalopt_report_t g;
    if (int r = scn_globalopt_solve(gopt.get(), kp.data(), &g)) return r;
    if (grep) *grep = g;
    if (!g.rejected && !kf_frame.empty()) {
      std::vector<scn_track_frame_t> tracked(res);
      const uint64_t S = gparams->submap_size;
      for (uint64_t f = 0; f < in.n_frames; ++f) {
        const int64_t k = kf_of_submap[f / S];
        if (res[f].lost || k < 0) continue;                                  // lost frames keep -inf
        if (kf_frame[k] == f) memcpy(res[f].cam2world, &kp[16 * k], 64);
        else propagate(tracked[kf_frame[k]].cam2world, &kp[16 * k], tracked[f].cam2world, res[f].cam2world);
      }
      reintegrate = out_ply != nullptr;
    }
  }
  for (uint64_t i = 0; i < in.n_frames; ++i)
    if (int r = scn_sens_set_pose(sp, i, res[i].cam2world)) return r;
  if (reintegrate) {                                 // a fresh volume through fuse's scene driver, at the poses just set
    scn_fuse_report_t fr;
    if (int r = scn::fuse_sens(sp, sens_path, out_ply, params, device, &fr)) return r;
    rep.mc_s = fr.mc_s; rep.ply_s = fr.ply_s;
    rep.mesh_vertices = fr.mesh_vertices; rep.mesh_faces = fr.mesh_faces;
  } else if (out_ply) {
    const double tm = now_s();
    float* xyz = nullptr; uint8_t* rgb = nullptr; uint32_t* tri = nullptr; uint64_t nV = 0, nF = 0;
    const int r = scn_tsdf_extract_mesh(vp, &xyz, &rgb, &tri, &nV, &nF);
    const scn::MallocPtr<float> o1(xyz); const scn::MallocPtr<uint8_t> o2(rgb); const scn::MallocPtr<uint32_t> o3(tri);
    if (r) return r;
    rep.mc_s = now_s() - tm;
    if (int q = scn_mesh_save_ply(out_ply, xyz, use_color ? rgb : nullptr, nV, tri, nF)) return q;
    rep.ply_s = now_s() - tm - rep.mc_s;
    rep.mesh_vertices = nV; rep.mesh_faces = nF;
  }
  const double ts = now_s();
  if (int r = scn_sens_save(sp, out_sens ? out_sens : sens_path)) return r;
  rep.sens_s = now_s() - ts;
  sens.reset();
  rep.total_s = now_s() - t_begin;
  return SCN_OK;
}

}  // namespace

extern "C" {

size_t scn_recons_report_sizeof(void) { return sizeof(scn_recons_report_t); }

int scn_recons_scene(const char* sens_path, const char* out_ply, const char* out_sens, const scn_tsdf_params* params,
                     const scn_track_params* tparams, int device, scn_recons_report_t* report) {
  if (!sens_path || !params || !tparams) return scn::fail(SCN_ERR_ARG, "null argument");
  scn_recons_report_t rep; memset(&rep, 0, sizeof(rep));
  const int rc = recons_scene(sens_path, out_ply, out_sens, params, tparams, nullptr, device, rep, nullptr);
  if (report) { rep.status = rc; *report = rep; }
  if (rc) { const std::string e = scn_last_error(); return scn::fail(rc, "%s: %s", sens_path, e.c_str()); }
  return SCN_OK;
}

int scn_recons_scene_global(const char* sens_path, const char* out_ply, const char* out_sens, const scn_tsdf_params* params,
                            const scn_track_params* tparams, const scn_globalopt_params* gparams, int device, scn_recons_report_t* report,
                            scn_globalopt_report_t* greport) {
  if (!sens_path || !params || !tparams || !gparams) return scn::fail(SCN_ERR_ARG, "null argument");
  scn_recons_report_t rep; memset(&rep, 0, sizeof(rep));
  scn_globalopt_report_t g; memset(&g, 0, sizeof(g));
  const int rc = recons_scene(sens_path, out_ply, out_sens, params, tparams, gparams, device, rep, &g);
  if (report) { rep.status = rc; *report = rep; }
  if (greport) *greport = g;
  if (rc) { const std::string e = scn_last_error(); return scn::fail(rc, "%s: %s", sens_path, e.c_str()); }
  return SCN_OK;
}

// `recons [--global] <params.txt> <params2.txt> <file.sens> [out.ply]`: <base>.ply beside the input unless an output is given; the
// trajectory is written back into the .sens.  --global: the keyframe trajectory is optimised and the stream re-integrated first.
int scn_recons_main(int argc, const char** argv) {
  std::vector<std::string> params; std::string sens, out;
  bool global = false;
  for (int i = 1; i < argc; ++i) {
    const std::string a = argv[i];
    if (a == "--global" && sens.empty() && params.empty()) global = true;
    else if (sens.empty() && a.size() > 5 && a.substr(a.size() - 5) == ".sens") sens = a;
    else if (!sens.empty()) out = a;
    else params.push_back(a);
  }
  if (sens.empty()) { printf("Usage: recons [--global] <params.txt> <params2.txt> <file.sens> [out.ply]\n"); return 255; }
  if (out.empty()) out = sens.substr(0, sens.size() - 5) + ".ply";
  scn_tsdf_params p; scn_tsdf_default_params(&p);
  p.voxel_size = 0.01f; p.trunc_base = 0.06f; p.trunc_scale = 0.02f;     // zParametersScanNet.txt:47-50 unless a file says otherwise
  scn_track_params tp; scn_track_default_params(&tp);
  scn_globalopt_params gp; scn_globalopt_default_params(&gp);
  for (const std::string& f : params)
    if (scn_tsdf_params_from_file(f.c_str(), &p) || scn_track_params_from_file(f.c_str(), &tp) ||
        (global && scn_globalopt_params_from_file(f.c_str(), &gp))) { fprintf(stderr, "%s\n", scn_last_error()); return 1; }
  printf("reconstructing %s: voxel %.4f m, truncation %.3f+%.3f*d, tracking at %ux%u\n", sens.c_str(), p.voxel_size, p.trunc_base, p.trunc_scale,
         tp.width, tp.height);
  scn_recons_report_t r;
  scn_globalopt_report_t g;
  const int rc = global ? scn_recons_scene_global(sens.c_str(), out.c_str(), nullptr, &p, &tp, &gp, 0, &r, &g)
                        : scn_recons_scene(sens.c_str(), out.c_str(), nullptr, &p, &tp, 0, &r);
  if (rc) { fprintf(stderr, "%s\n", scn_last_error()); return 1; }
  printf("tracked %llu of %llu frames (%llu lost) in %.3f s = %.1f frames/s incl. decode; %llu blocks\n", (unsigned long long)r.frames_tracked,
         (unsigned long long)r.frames, (unsigned long long)r.frames_lost, r.recons_s, r.frames / std::max(r.recons_s, 1e-9),
         (unsigned long long)r.blocks_allocated);
  if (global)
    printf("global optimisation: %u keyframes, %u consecutive + %u loop edges, %u removed, %s; RMS %.2f -> %.2f mm\n", g.keyframes,
           g.edges_consecutive, g.edges_loop, g.edges_removed, g.rejected ? "rejected (tracked trajectory kept)" : "accepted",
           g.rms_before * 1e3, g.rms_after * 1e3);
  printf("mesh written to %s with %llu vertices, %llu faces; trajectory written to %s\n", out.c_str(), (unsigned long long)r.mesh_vertices,
         (unsigned long long)r.mesh_faces, sens.c_str());
  return 0;
}

}  // extern "C"
