// `freespace` — the free-space stage of the reference pipeline in library form (DESIGN.md §6h):
//   <exe> <file.sens>                                   (Server/scan_processor.py:150-152, Server/config/scan_stages.json:43-47)
//   <exe> [params.txt] <file.sens> [out.grid] [--voxel V]
// Reads every pose of the .sens stream, derives the lattice box the frames can observe, inflates the depth of the frames that
// have a pose on the GPU (scn::sens_depth_to_device) chunk by chunk, counts free / occupied observations per voxel
// (scn_freespace_integrate_device), crops to the labelled voxels and writes `<base>.grid`.
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "scn_common.h"

namespace {

using scn::now_s;
constexpr uint32_t kChunk = 1024;            // frames decoded per scn::sens_depth_to_device call

}  // namespace

extern "C" {

int scn_freespace_save_grid(const char* path, float voxel_size, const int32_t lo[3], const uint64_t dims[3], const uint8_t* labels) {
  if (!path || !lo || !dims) return scn::fail(SCN_ERR_ARG, "null argument");
  const uint64_t n = dims[0] * dims[1] * dims[2];
  if (n && !labels) return scn::fail(SCN_ERR_ARG, "null labels");
  FILE* f = fopen(path, "wb");
  if (!f) return scn::fail(SCN_ERR_IO, "cannot open %s for writing", path);
  unsigned char hdr[52];
  const uint32_t version = 1;
  memcpy(hdr, "SCNGRID\0", 8);
  memcpy(hdr + 8, &version, 4);
  memcpy(hdr + 12, &voxel_size, 4);
  memcpy(hdr + 16, dims, 24);
  memcpy(hdr + 40, lo, 12);                                      // little-endian host (x86-64, aarch64)
  bool ok = fwrite(hdr, 1, sizeof(hdr), f) == sizeof(hdr) && (n == 0 || fwrite(labels, 1, n, f) == n);
  ok = (fclose(f) == 0) && ok;
  if (!ok) return scn::fail(SCN_ERR_IO, "write to %s failed", path);
  return SCN_OK;
}

int scn_freespace_scene(const char* sens_path, const char* out_grid, const scn_freespace_params* params, int device,
                        scn_freespace_report_t* report) {
  if (!sens_path || !params) return scn::fail(SCN_ERR_ARG, "null argument");
  const double t_begin = now_s();
  scn_sens* sp = nullptr;
  if (int rc = scn_sens_open(sens_path, &sp)) return rc;
  const scn::SensPtr s(sp);
  scn_sens_info_t in;
  if (int rc = scn_sens_info(s.get(), &in)) return rc;
  if (in.depth_compression != 0 && in.depth_compression != 1)
    return scn::fail(SCN_ERR_UNSUPPORTED, "%s: depth compression %d (only raw and zlib u16 are decoded)", sens_path, in.depth_compression);
  // 1. the frames that have a pose, and their poses (no decode)
  scn::PosedFrames plan;
  if (int rc = scn::posed_frames(s.get(), 0, in.n_frames, plan)) return rc;
  const uint32_t n_posed = (uint32_t)plan.frames.size();
  // 2. the envelope, the handle
  int32_t lo[3]; uint64_t dims[3];
  if (int rc = scn_freespace_envelope(plan.poses.data(), n_posed, in.depth_intrinsic, in.depth_width, in.depth_height, params, lo, dims)) return rc;
  scn_freespace* hp = nullptr;
  if (int rc = scn_freespace_create(params, in.depth_width, in.depth_height, in.depth_shift, lo, dims, device, &hp)) return rc;
  const scn::FreespacePtr h(hp);
  // 3. those frames chunk by chunk: decoded into device memory, counted
  const size_t px = (size_t)in.depth_width * in.depth_height;
  scn::HandleStreamPtr stream;
  if (int rc = scn::create(stream)) return rc;
  const scn::DevicePtr<uint16_t> d_depth(n_posed ? (uint16_t*)scn_device_alloc((size_t)kChunk * px * 2) : nullptr);
  if (n_posed && !d_depth)
    return scn::fail(SCN_ERR_CUDA, "cannot allocate %zu bytes of depth frames", (size_t)kChunk * px * 2);
  double decode_s = 0;
  for (uint32_t i0 = 0; i0 < n_posed; i0 += kChunk) {
    const uint32_t n = std::min(kChunk, n_posed - i0);
    const double td0 = now_s();
    if (int rc = scn::sens_depth_to_device(s.get(), &plan.frames[i0], n, d_depth.get(), stream.get())) return rc;
    decode_s += now_s() - td0;
    if (int rc = scn_freespace_integrate_device(h.get(), n, d_depth.get(), &plan.poses[(size_t)i0 * 16], in.depth_intrinsic)) return rc;
  }
  // 4. labels of the crop box, the file
  int32_t olo[3]; uint64_t od[3];
  uint8_t* lp = nullptr;
  if (int r = scn_freespace_download(h.get(), olo, od, &lp, nullptr, nullptr)) return r;
  const scn::MallocPtr<uint8_t> labels(lp);
  double write_s = 0;
  if (out_grid) {
    const double tw0 = now_s();
    if (int r = scn_freespace_save_grid(out_grid, params->voxel_size, olo, od, labels.get())) return r;
    write_s = now_s() - tw0;
  }
  scn_freespace_report_t rep;
  if (int r = scn_freespace_handle_report(h.get(), &rep)) return r;
  rep.frames_skipped_pose = in.n_frames - rep.frames_used;
  rep.decode_s = decode_s; rep.write_s = write_s;
  rep.total_s = now_s() - t_begin;
  if (report) *report = rep;
  return SCN_OK;
}

int scn_freespace_main(int argc, const char** argv) {
  std::vector<std::string> pos;
  float voxel = 0.f;
  for (int i = 1; i < argc; ++i) {
    const std::string a = argv[i];
    if (a == "--voxel" && i + 1 < argc) { voxel = (float)atof(argv[++i]); if (!(voxel > 0.f)) { fprintf(stderr, "freespace: --voxel needs a size > 0\n"); return 255; } continue; }
    pos.push_back(a);
  }
  auto is_sens = [](const std::string& s) { return s.size() > 5 && s.compare(s.size() - 5, 5, ".sens") == 0; };
  std::string params_path, sens, out;
  if (pos.size() == 1) sens = pos[0];
  else if (pos.size() == 2 && is_sens(pos[0])) { sens = pos[0]; out = pos[1]; }
  else if (pos.size() == 2) { params_path = pos[0]; sens = pos[1]; }
  else if (pos.size() == 3) { params_path = pos[0]; sens = pos[1]; out = pos[2]; }
  if (sens.empty()) {
    printf("Usage: freespace [params.txt] <file.sens> [out.grid] [--voxel V]\n"
           "       writes <base>.grid beside the input: 0 unknown, 1 free, 2 occupied per voxel (DESIGN.md §6h)\n");
    return 255;
  }
  scn_freespace_params p; scn_freespace_default_params(&p);
  if (!params_path.empty()) {
    // only the depth range and the maximum integration distance are taken from a reconstruction parameter file
    scn_tsdf_params tp; scn_tsdf_default_params(&tp);
    tp.depth_min = p.depth_min; tp.depth_max = p.depth_max; tp.max_integration_distance = p.max_distance;
    if (scn_tsdf_params_from_file(params_path.c_str(), &tp)) { fprintf(stderr, "freespace: %s\n", scn_last_error()); return 1; }
    p.depth_min = tp.depth_min; p.depth_max = tp.depth_max; p.max_distance = tp.max_integration_distance;
  }
  if (voxel > 0.f) p.voxel_size = p.band_base = voxel;
  if (out.empty()) out = (is_sens(sens) ? sens.substr(0, sens.size() - 5) : sens) + ".grid";
  scn_freespace_report_t r;
  if (scn_freespace_scene(sens.c_str(), out.c_str(), &p, 0, &r)) { fprintf(stderr, "freespace: %s\n", scn_last_error()); return 1; }
  printf("freespace %s: %llu frames (%llu without pose), voxel %.4f m, envelope %llux%llux%llu -> grid %llux%llux%llu at (%d, %d, %d): "
         "%llu free, %llu occupied, %llu unknown; %.3f s -> %s\n",
         sens.c_str(), (unsigned long long)r.frames_used, (unsigned long long)r.frames_skipped_pose, p.voxel_size,
         (unsigned long long)r.envelope_dims[0], (unsigned long long)r.envelope_dims[1], (unsigned long long)r.envelope_dims[2],
         (unsigned long long)r.output_dims[0], (unsigned long long)r.output_dims[1], (unsigned long long)r.output_dims[2],
         r.output_lo[0], r.output_lo[1], r.output_lo[2], (unsigned long long)r.voxels_free, (unsigned long long)r.voxels_occupied,
         (unsigned long long)r.voxels_unknown, r.total_s, out.c_str());
  return 0;
}

}  // extern "C"
