// `freespace` — the free-space stage of the reference pipeline in library form (DESIGN.md §6h):
//   <exe> <file.sens>                                   (Server/scan_processor.py:150-152, Server/config/scan_stages.json:43-47)
//   <exe> [params.txt] <file.sens> [out.grid] [--voxel V]
// Reads every pose of the .sens stream, derives the lattice box the frames can observe, inflates the depth of the frames that
// have a pose on the GPU (scn_inflate_batch_device) chunk by chunk, counts free / occupied observations per voxel
// (scn_freespace_integrate_device), crops to the labelled voxels and writes `<base>.grid`.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "scn_common.h"

namespace {

double now_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

constexpr uint32_t kChunk = 1024;            // frames decoded per scn_inflate_batch_device call

// owners of the C-ABI resources the driver holds
struct Sens { scn_sens* s = nullptr; ~Sens() { scn_sens_close(s); } };
struct Handle { scn_freespace* h = nullptr; ~Handle() { scn_freespace_destroy(h); } };
struct DevBuf { void* p = nullptr; ~DevBuf() { scn_device_free(p); } };
template <class T> struct Owned { T* p = nullptr; ~Owned() { scn_free(p); } };

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
  Sens s;
  if (int rc = scn_sens_open(sens_path, &s.s)) return rc;
  scn_sens_info_t in;
  if (int rc = scn_sens_info(s.s, &in)) return rc;
  if (in.depth_compression != 0 && in.depth_compression != 1)
    return scn::fail(SCN_ERR_UNSUPPORTED, "%s: depth compression %d (only raw and zlib u16 are decoded)", sens_path, in.depth_compression);
  // 1. every pose (no decode)
  std::vector<float> poses((size_t)in.n_frames * 16);
  for (uint64_t f = 0; f < in.n_frames; ++f)
    if (int rc = scn_sens_frame_meta(s.s, f, &poses[f * 16], nullptr, nullptr, nullptr, nullptr)) return rc;   // never a zero pose taken as valid
  // 2. the envelope, the handle
  int32_t lo[3]; uint64_t dims[3];
  if (int rc = scn_freespace_envelope(poses.data(), (uint32_t)in.n_frames, in.depth_intrinsic, in.depth_width, in.depth_height, params, lo, dims)) return rc;
  Handle h;
  if (int rc = scn_freespace_create(params, in.depth_width, in.depth_height, in.depth_shift, lo, dims, device, &h.h)) return rc;
  // 3. per chunk: the frames with a pose, compacted (a frame without one is never decoded: sensorData.h:382), decoded into
  //    device memory, counted
  const size_t px = (size_t)in.depth_width * in.depth_height;
  DevBuf d_depth;
  void* stream = nullptr;
  double decode_s = 0;
  std::vector<const uint8_t*> src; std::vector<uint64_t> len; std::vector<float> cp;
  int rc = 0;
  if (scn_stream_create(&stream)) return SCN_ERR_CUDA;
  for (uint64_t f0 = 0; f0 < in.n_frames && !rc; f0 += kChunk) {
    const uint64_t f1 = std::min<uint64_t>(in.n_frames, f0 + kChunk);
    src.clear(); len.clear(); cp.clear();
    for (uint64_t f = f0; f < f1; ++f) {
      if (poses[f * 16] == -INFINITY) continue;
      const uint8_t* cpay = nullptr; const uint8_t* dpay = nullptr; uint64_t db = 0;
      if ((rc = scn_sens_frame_payload(s.s, f, &cpay, &dpay)) || (rc = scn_sens_frame_meta(s.s, f, nullptr, nullptr, nullptr, nullptr, &db))) break;
      src.push_back(dpay); len.push_back(db);
      cp.insert(cp.end(), &poses[f * 16], &poses[f * 16] + 16);
    }
    const uint32_t n = (uint32_t)src.size();
    if (rc) break;
    if (!n) continue;
    if (!d_depth.p && !(d_depth.p = scn_device_alloc((size_t)kChunk * px * 2))) { rc = scn::fail(SCN_ERR_CUDA, "cannot allocate %zu bytes of depth frames", (size_t)kChunk * px * 2); break; }
    const double td0 = now_s();
    if (in.depth_compression == 1) {
      rc = scn_inflate_batch_device(src.data(), len.data(), n, (uint64_t)px * 2, d_depth.p, stream);
    } else {
      for (uint32_t i = 0; i < n && !rc; ++i) {
        if (len[i] < px * 2) { rc = scn::fail(SCN_ERR_FORMAT, "%s: raw depth payload of %llu bytes, need %zu", sens_path, (unsigned long long)len[i], px * 2); break; }
        rc = scn_memcpy_h2d((uint16_t*)d_depth.p + (size_t)i * px, src[i], px * 2, stream);
      }
    }
    decode_s += now_s() - td0;
    if (!rc) rc = scn_freespace_integrate_device(h.h, n, (const uint16_t*)d_depth.p, cp.data(), in.depth_intrinsic);
  }
  scn_stream_destroy(stream);
  if (rc) return rc;
  // 4. labels of the crop box, the file
  int32_t olo[3]; uint64_t od[3];
  Owned<uint8_t> labels;
  if (int r = scn_freespace_download(h.h, olo, od, &labels.p, nullptr, nullptr)) return r;
  double write_s = 0;
  if (out_grid) {
    const double tw0 = now_s();
    if (int r = scn_freespace_save_grid(out_grid, params->voxel_size, olo, od, labels.p)) return r;
    write_s = now_s() - tw0;
  }
  scn_freespace_report_t rep;
  if (int r = scn_freespace_handle_report(h.h, &rep)) return r;
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
