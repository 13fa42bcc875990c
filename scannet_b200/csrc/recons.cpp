// `recons` — the reconstruction stage of the reference pipeline in library form:
//   FriedLiver.exe <params.txt> <params2.txt> <file.sens>          (Server/scan_processor.py:27-29,123-126)
// Every frame of the stream is decoded on the GPU (depth by the inflate kernel, colour by the device JPEG decoder registered to
// the depth image, as `fuse` does), tracked against the model and integrated at its tracked pose (csrc/track.cu, DESIGN.md §6j);
// then marching cubes -> <base>.ply and the trajectory -> the .sens (s_overwriteOrigSensTrajectory, zParametersScanNet.txt:5):
// only the 64-byte pose fields change, the payloads are written back byte for byte.  Nothing is written when a call fails.
// Not BundleFusion: no sparse features, no global optimisation (the trajectory is a frame-to-model tracker's).
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

constexpr uint32_t kChunk = 256;                    // frames decoded per call of the depth and colour decoders

int recons_scene(const char* sens_path, const char* out_ply, const char* out_sens, const scn_tsdf_params* params,
                 const scn_track_params* tparams, int device, scn_recons_report_t& rep) {
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
  }
  rep.recons_s = now_s() - t0;
  for (const scn_track_frame_t& r : res) rep.frames_lost += r.lost;
  rep.frames_tracked = in.n_frames - rep.frames_lost;
  scn_track_phase_ms(tp, &rep.filter_pyramid_ms, &rep.icp_ms, &rep.integrate_ms, &rep.raycast_ms);
  scn_track_stats(tp, nullptr, &rep.kernel_launches);
  scn_tsdf_stats_t st; scn_tsdf_stats(vp, &st);
  rep.blocks_allocated = st.blocks_allocated;
  if (out_ply) {
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
  for (uint64_t i = 0; i < in.n_frames; ++i)
    if (int r = scn_sens_set_pose(sp, i, res[i].cam2world)) return r;
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
  const int rc = recons_scene(sens_path, out_ply, out_sens, params, tparams, device, rep);
  if (report) { rep.status = rc; *report = rep; }
  if (rc) { const std::string e = scn_last_error(); return scn::fail(rc, "%s: %s", sens_path, e.c_str()); }
  return SCN_OK;
}

// `recons <params.txt> <params2.txt> <file.sens> [out.ply]`: <base>.ply beside the input unless an output is given; the trajectory
// is written back into the .sens.
int scn_recons_main(int argc, const char** argv) {
  std::vector<std::string> params; std::string sens, out;
  for (int i = 1; i < argc; ++i) {
    const std::string a = argv[i];
    if (sens.empty() && a.size() > 5 && a.substr(a.size() - 5) == ".sens") sens = a;
    else if (!sens.empty()) out = a;
    else params.push_back(a);
  }
  if (sens.empty()) { printf("Usage: recons <params.txt> <params2.txt> <file.sens> [out.ply]\n"); return 255; }
  if (out.empty()) out = sens.substr(0, sens.size() - 5) + ".ply";
  scn_tsdf_params p; scn_tsdf_default_params(&p);
  p.voxel_size = 0.01f; p.trunc_base = 0.06f; p.trunc_scale = 0.02f;     // zParametersScanNet.txt:47-50 unless a file says otherwise
  scn_track_params tp; scn_track_default_params(&tp);
  for (const std::string& f : params)
    if (scn_tsdf_params_from_file(f.c_str(), &p) || scn_track_params_from_file(f.c_str(), &tp)) { fprintf(stderr, "%s\n", scn_last_error()); return 1; }
  printf("reconstructing %s: voxel %.4f m, truncation %.3f+%.3f*d, tracking at %ux%u\n", sens.c_str(), p.voxel_size, p.trunc_base, p.trunc_scale,
         tp.width, tp.height);
  scn_recons_report_t r;
  if (scn_recons_scene(sens.c_str(), out.c_str(), nullptr, &p, &tp, 0, &r)) { fprintf(stderr, "%s\n", scn_last_error()); return 1; }
  printf("tracked %llu of %llu frames (%llu lost) in %.3f s = %.1f frames/s incl. decode; %llu blocks\n", (unsigned long long)r.frames_tracked,
         (unsigned long long)r.frames, (unsigned long long)r.frames_lost, r.recons_s, r.frames / std::max(r.recons_s, 1e-9),
         (unsigned long long)r.blocks_allocated);
  printf("mesh written to %s with %llu vertices, %llu faces; trajectory written to %s\n", out.c_str(), (unsigned long long)r.mesh_vertices,
         (unsigned long long)r.mesh_faces, sens.c_str());
  return 0;
}

}  // extern "C"
