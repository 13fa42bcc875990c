// `fuse` — the reconstruction stage contract of the reference pipeline in library form:
//   <exe> <params.txt> [<params2.txt>] <file.sens> [out.ply]        (Server/scan_processor.py:27-35,123-138)
//   <exe> --gpus N <params.txt> ... <a.sens> <b.sens> ...           one scene per GPU at a time (Server/process.py:75 serialises
//                                                                   one scan per GPU; here N scans run on N GPUs, SURVEY.md §8e)
// Reads the .sens stream (SensReader), fuses every frame that has a valid pose into the hashed TSDF volume (poses come from
// the file: camera tracking / bundle adjustment is not part of this path), extracts the surface with marching cubes and
// writes `<base>_vh.ply` in the VCGLIB layout the `segment` stage reads (Server/config/scan_stages.json:33-37).
//
// Decode.  Default ("gpu"): the COMPRESSED payloads are uploaded and decoded in HBM — depth by the inflate kernel
// (csrc/inflate.cu), JPEG colour by the device JPEG decoder (csrc/jpeg_gpu.cu), which samples only the colour pixels the
// depth image needs — in chunks of a few hundred frames, two decoder threads (depth, colour) one chunk ahead of the
// integration, so no raw frame crosses PCIe or touches a host core.  "host" (SCN_FUSE_DECODE=host; automatic for PNG / raw
// colour): a host thread pool inflates / decodes one chunk ahead and the frames are handed over in pinned memory.
#include <atomic>
#include <condition_variable>
#include <functional>
#include <memory>
#include <mutex>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

#include "scn_common.h"
#include "stage_pool.h"

namespace {

// Persistent worker pool: run(fn) executes fn() on every worker and on the caller, and returns when all are done
// (spawning 64 threads per 128-frame chunk cost ~3 ms of a ~10 ms chunk).
class Pool {
 public:
  explicit Pool(unsigned workers) { for (unsigned i = 0; i < workers; ++i) th_.emplace_back([this]() { loop(); }); }
  ~Pool() { { std::lock_guard<std::mutex> l(m_); stop_ = true; ++gen_; } cv_.notify_all(); for (auto& t : th_) t.join(); }
  void run(const std::function<void()>& fn) {
    { std::lock_guard<std::mutex> l(m_); fn_ = &fn; pending_ = (unsigned)th_.size(); ++gen_; }
    cv_.notify_all();
    fn();
    std::unique_lock<std::mutex> l(m_); done_.wait(l, [this]() { return pending_ == 0; });
  }
 private:
  void loop() {
    unsigned long seen = 0;
    for (;;) {
      const std::function<void()>* fn;
      { std::unique_lock<std::mutex> l(m_); cv_.wait(l, [&]() { return gen_ != seen; }); seen = gen_; if (stop_) return; fn = fn_; }
      (*fn)();
      { std::lock_guard<std::mutex> l(m_); if (--pending_ == 0) done_.notify_one(); }
    }
  }
  std::vector<std::thread> th_; std::mutex m_; std::condition_variable cv_, done_;
  const std::function<void()>* fn_ = nullptr; unsigned pending_ = 0; unsigned long gen_ = 0; bool stop_ = false;
};

struct Chunk { scn::PinnedPtr<uint16_t> depth; scn::PinnedPtr<uint8_t> rgb; std::vector<float> poses; uint32_t n = 0; };

// The first call of a scene that failed, on whichever thread: its code, and its text, read on that thread (scn_last_error is
// per thread).
struct FirstFailure {
  std::atomic<int> rc{0}; std::mutex m; std::string err;
  void set(int code) { std::lock_guard<std::mutex> l(m); if (!rc.load()) { err = scn_last_error(); rc.store(code); } }
  explicit operator bool() const { return rc.load() != 0; }
};

using scn::now_s;

void decode_chunk(const scn_sens* s, const scn_sens_info_t& in, const std::vector<int32_t>& lut, bool use_color, uint64_t f0, uint32_t n, Chunk& c, Pool& pool,
                  FirstFailure& fail) {
  const size_t px = (size_t)in.depth_width * in.depth_height;
  c.n = n; c.poses.assign((size_t)n * 16, 0.f);
  std::atomic<uint32_t> next{0};
  pool.run([&]() {
    static thread_local std::vector<uint8_t> col;                               // kept per pool thread: no 1-4 MB allocation per chunk
    col.resize(use_color ? (size_t)in.color_width * in.color_height * 3 : 0);
    for (uint32_t i; (i = next.fetch_add(1)) < n && !fail;) {
      float* T = &c.poses[(size_t)i * 16];
      int r = scn_sens_frame_meta(s, f0 + i, T, nullptr, nullptr, nullptr, nullptr);
      if (!r && T[0] != -INFINITY) {                                             // a frame without a pose is skipped by the integrator
        r = scn_sens_frame_depth_u16(s, f0 + i, c.depth.get() + (size_t)i * px);
        if (!r && use_color) r = scn::sens_color_to_depth(s, f0 + i, lut.data(), px, col.data(), c.rgb.get() + (size_t)i * px * 3);
      }
      if (r) fail.set(r);
    }
  });
}

// ---- one scene on one GPU ------------------------------------------------------------------------------------------------------
struct SceneJob {
  std::string sens_path, out_path;          // out_path empty = no mesh
  scn_tsdf_params params;                   // width / height / depth_shift are taken from the stream
  int device = 0;
  bool verbose = true;
  const char* decode_mode = nullptr;        // "gpu", "host" or null (automatic)
};

// The volume (16 GiB of voxel blocks with the CLI's defaults: cudaMalloc + first clear + cudaFree cost 0.15-0.4 s, as much as
// fusing a 5,578-frame scan; a reset clears only the used blocks in a few ms) is kept per device from one scene to the next - by
// the workers of scn_fuse_many and by consecutive scn_fuse_scene calls of a process alike; scn_release_cached_staging frees it.
struct VolSlot {
  int device = 0;
  scn_tsdf* vol = nullptr; scn_tsdf_params p;
  void release() { if (vol) scn_tsdf_destroy(vol); vol = nullptr; }
};
// The double-buffered frame arrays of the GPU-decode mode (3 GB at 1024-frame chunks with colour) come from a per-device pool
// like the decoders' staging: allocating and freeing them per scene cost up to 0.2 s (cudaFree synchronises the device).
struct FrameBufs {
  int device = 0;
  void* buf[4] = {nullptr, nullptr, nullptr, nullptr}; size_t cap[4] = {0, 0, 0, 0};       // depth x2, colour x2
  void* take(int i, size_t bytes) {
    if (bytes > cap[i]) { scn_device_free(buf[i]); buf[i] = scn_device_alloc(bytes); cap[i] = buf[i] ? bytes : 0; }
    return buf[i];
  }
  void release() { for (int i = 0; i < 4; ++i) { scn_device_free(buf[i]); buf[i] = nullptr; cap[i] = 0; } }
};
scn::StagePool<FrameBufs>& frame_pool() { static auto* p = new scn::StagePool<FrameBufs>(); return *p; }
scn::StagePool<VolSlot>& vol_pool() { static auto* p = new scn::StagePool<VolSlot>(); return *p; }

int fuse_open_scene(const SceneJob& job, const scn_sens* s, scn_fuse_report_t& rep, double t_begin);

int fuse_scene(const SceneJob& job, scn_fuse_report_t* rep_out) {
  scn_fuse_report_t rep; memset(&rep, 0, sizeof(rep));
  rep.device = job.device;
  const double t_begin = now_s();
  if (scn_set_device(job.device)) return SCN_ERR_CUDA;
  std::thread warm([dev = job.device]() { scn_set_device(dev); scn_cuda_warmup(); });          // context creation overlaps reading the .sens file
  scn_sens* sp = nullptr;
  const int open_rc = scn_sens_open(job.sens_path.c_str(), &sp);
  const std::string open_err = open_rc ? scn_last_error() : "";
  warm.join();
  if (open_rc) return scn::fail(open_rc, "%s", open_err.c_str());
  scn::SensPtr sens(sp);
  const int rc = fuse_open_scene(job, sens.get(), rep, t_begin);
  sens.reset();                                                // total_s includes unmapping the file
  rep.total_s = now_s() - t_begin;
  if (rep_out) *rep_out = rep;
  return rc;
}

// The scene of an open stream, with the poses it holds in memory: the volume, the decode and the integration, then the mesh.
int fuse_open_scene(const SceneJob& job, const scn_sens* s, scn_fuse_report_t& rep, double t_begin) {
  scn_sens_info_t in; scn_sens_info(s, &in);
  scn_tsdf_params p = job.params;
  p.width = in.depth_width; p.height = in.depth_height; p.depth_shift = in.depth_shift;   // integrate at the stream's depth resolution
  if (p.batch_frames == 0) p.batch_frames = 32;
  const bool use_color = in.color_compression <= 2 && in.color_width > 0 && in.color_height > 0;   // raw, PNG, JPEG (sensorData.h:600-616)
  if (job.verbose)
    printf("fusing %s: %llu frames %ux%u, voxel %.4f m, truncation %.3f+%.3f*d\n", job.sens_path.c_str(), (unsigned long long)in.n_frames, in.depth_width,
           in.depth_height, p.voxel_size, p.trunc_base, p.trunc_scale);
  scn_tsdf* vol = nullptr;
  scn::StagePool<VolSlot>::Lease vs(vol_pool());
  if (vs->vol && !memcmp(&vs->p, &p, sizeof(p))) {                                     // same volume layout as the previous scene on this GPU
    vol = vs->vol;
    if (int r = scn_tsdf_reset(vol)) { const std::string e = scn_last_error(); vs->release(); return scn::fail(r, "%s: %s", job.sens_path.c_str(), e.c_str()); }
    rep.volume_reused = 1;
  } else {
    vs->release();
    if (int r = scn_tsdf_create(&p, job.device, &vol)) return scn::fail(r, "%s: %s", job.sens_path.c_str(), scn_last_error());
    vs->vol = vol; vs->p = p;
  }
  const size_t px = (size_t)in.depth_width * in.depth_height;
  std::vector<int32_t> lut; if (use_color) scn::build_color_lut(in, lut);
  // decode mode
  const bool gpu_able = in.depth_compression == 0 || in.depth_compression == 1;
  const bool gpu_decode = gpu_able && !(job.decode_mode && !strcmp(job.decode_mode, "host"));
  if (job.verbose)
    printf("decode: %s\n", !gpu_decode ? "host thread pool" : (use_color && in.color_compression != 2) ? "GPU inflate (depth), host thread pool (raw / PNG colour)"
                                                                                      : "GPU inflate (depth) + GPU JPEG (colour), compressed payloads uploaded");
  rep.gpu_decode = gpu_decode ? 1 : 0;
  const double t0 = now_s();
  rep.setup_s = t0 - t_begin;
  FirstFailure fail;
  double tt0 = 0;                                  // GPU decode: start of the teardown, which ends when the decode buffers are released
  if (gpu_decode) {
    const char* ce = getenv("SCN_FUSE_CHUNK");
    const uint32_t CH = (uint32_t)std::max(16, std::min(4096, ce ? atoi(ce) : 1024));   // frames per decode chunk: enough streams in flight for the one-warp-per-frame decoders
    const uint64_t n_chunks = (in.n_frames + CH - 1) / CH;
    uint16_t* d_depth[2] = {nullptr, nullptr}; uint8_t* d_rgb[2] = {nullptr, nullptr};
    scn::DevicePtr<int32_t> d_lut; scn::HandleStreamPtr st_d, st_c; scn::PinnedPtr<uint8_t> h_rgb;
    scn::StagePool<FrameBufs>::Lease fb(frame_pool());
    for (int b = 0; b < 2; ++b) {
      d_depth[b] = (uint16_t*)fb->take(b, (size_t)CH * px * 2);
      if (use_color) d_rgb[b] = (uint8_t*)fb->take(2 + b, (size_t)CH * px * 3);
      if (!d_depth[b] || (use_color && !d_rgb[b])) fail.set(SCN_ERR_CUDA);
    }
    if (use_color && !fail) {
      d_lut.reset((int32_t*)scn_device_alloc(px * 4));
      if (int r = d_lut ? scn_memcpy_h2d(d_lut.get(), lut.data(), px * 4, nullptr) : SCN_ERR_CUDA) fail.set(r);
    }
    if (!fail) { int r = scn::create(st_d); if (!r) r = scn::create(st_c); if (r) fail.set(r); }
    rep.buffers_s = now_s() - t0;
    std::mutex m; std::condition_variable cv;
    std::vector<int> depth_done(n_chunks, 0), color_done(n_chunks, 0);            // 1 = ready, -1 = failed
    std::vector<scn::PosedFrames> plan(n_chunks);
    uint64_t consumed = 0;                                                          // chunks whose buffers are free again
    bool stop = false;
    for (uint64_t c = 0; c < n_chunks && !fail; ++c) {
      const uint64_t f0 = c * CH, f1 = std::min<uint64_t>(in.n_frames, f0 + CH);
      if (int r = scn::posed_frames(s, f0, f1, plan[c])) fail.set(r);
      else rep.frames_skipped_pose += (f1 - f0) - plan[c].frames.size();
    }
    std::unique_ptr<Pool> color_pool;
    if (use_color && in.color_compression != 2) color_pool.reset(new Pool(std::max(1u, std::min(32u, std::thread::hardware_concurrency())) - 1));
    auto decoder = [&](bool is_color) {
      scn_set_device(job.device);
      std::vector<const uint8_t*> src; std::vector<uint64_t> len;
      for (uint64_t c = 0; c < n_chunks; ++c) {
        { std::unique_lock<std::mutex> l(m); cv.wait(l, [&]() { return stop || c < consumed + 2; }); if (stop) return; }
        const scn::PosedFrames& pl = plan[c];
        const uint32_t n = (uint32_t)pl.frames.size();
        int r = 0;
        if (n) {
          const double td0 = now_s();
          if (!is_color) {
            r = scn::sens_depth_to_device(s, pl.frames.data(), n, d_depth[c & 1], st_d.get());
            double ps = 0, km = 0; scn_inflate_last_timings(&ps, &km, nullptr, nullptr);
            if (!r) { std::lock_guard<std::mutex> l(m); rep.depth_decode_s += now_s() - td0; rep.depth_pack_s += ps; rep.depth_kernel_s += km * 1e-3; }
          } else if (in.color_compression != 2) {
            // raw / PNG colour: host pool into a pinned chunk (registered to depth on the way), one upload
            if (!h_rgb) h_rgb.reset((uint8_t*)scn_host_alloc((size_t)CH * px * 3));
            if (!h_rgb) r = SCN_ERR_CUDA;
            std::atomic<uint32_t> nx{0};
            if (!r) color_pool->run([&]() {
              static thread_local std::vector<uint8_t> col;
              col.resize((size_t)in.color_width * in.color_height * 3);
              for (uint32_t i; (i = nx.fetch_add(1)) < n && !fail;)
                if (int q = scn::sens_color_to_depth(s, pl.frames[i], lut.data(), px, col.data(), h_rgb.get() + (size_t)i * px * 3)) fail.set(q);
            });
            if (!r) r = fail.rc.load();                                           // the scene failed (here or elsewhere): no upload
            if (!r) r = scn_memcpy_h2d(d_rgb[c & 1], h_rgb.get(), (size_t)n * px * 3, st_c.get());
            if (!r) { std::lock_guard<std::mutex> l(m); rep.color_decode_s += now_s() - td0; }
          } else {
            src.resize(n); len.resize(n);
            for (uint32_t i = 0; i < n && !r; ++i)
              if (!(r = scn_sens_frame_payload(s, pl.frames[i], &src[i], nullptr))) r = scn_sens_frame_meta(s, pl.frames[i], nullptr, nullptr, nullptr, &len[i], nullptr);
            uint32_t k = 0;
            if (!r) r = scn_jpeg_decode_batch_device(src.data(), len.data(), n, in.color_width, in.color_height, d_lut.get(), (uint32_t)px, d_rgb[c & 1], st_c.get(), &k);
            double hs = 0, em = 0, cm = 0; scn_jpeg_last_timings(&hs, &em, &cm);
            if (!r) { std::lock_guard<std::mutex> l(m); rep.color_frames_on_device += k; rep.color_decode_s += now_s() - td0;
                      rep.color_host_s += hs; rep.color_entropy_s += em * 1e-3; rep.color_convert_s += cm * 1e-3; }
          }
        }
        if (r) fail.set(r);
        { std::lock_guard<std::mutex> l(m); (is_color ? color_done : depth_done)[c] = r ? -1 : 1; }
        cv.notify_all();
        if (r) return;
      }
    };
    std::thread th_d, th_c;
    if (!fail) { th_d = std::thread(decoder, false); if (use_color) th_c = std::thread(decoder, true); }
    for (uint64_t c = 0; c < n_chunks && !fail; ++c) {
      const double tw0 = now_s();
      {
        std::unique_lock<std::mutex> l(m);
        cv.wait(l, [&]() { return depth_done[c] != 0 && (!use_color || color_done[c] != 0); });
        if (depth_done[c] < 0 || (use_color && color_done[c] < 0)) break;
      }
      rep.decode_wait_s += now_s() - tw0;
      const scn::PosedFrames& pl = plan[c];
      if (!pl.frames.empty()) {
        const double ti0 = now_s();
        if (int r = scn_tsdf_integrate_device(vol, (uint32_t)pl.frames.size(), d_depth[c & 1], use_color ? d_rgb[c & 1] : nullptr, pl.poses.data(), in.depth_intrinsic)) { fail.set(r); break; }
        if (int r = scn_tsdf_sync(vol)) { fail.set(r); break; }                         // the buffers of this chunk may be overwritten now
        rep.integrate_s += now_s() - ti0;
      }
      { std::lock_guard<std::mutex> l(m); consumed = c + 1; }
      cv.notify_all();
    }
    tt0 = now_s();
    { std::lock_guard<std::mutex> l(m); stop = true; }
    cv.notify_all();
    if (th_d.joinable()) th_d.join();
    if (th_c.joinable()) th_c.join();
  } else {
    // host decode is the bottleneck of this mode (one frame = ~2 ms inflate + ~1-3 ms JPEG on one core): up to 64 cores,
    // chunks of two frames per worker
    const unsigned threads = std::max(1u, std::min(64u, std::thread::hardware_concurrency()));
    const uint32_t CH = std::max(32u, 2 * threads);
    Pool pool(threads - 1);
    Chunk ch[2];
    for (Chunk& c : ch) {
      c.depth.reset((uint16_t*)scn_host_alloc(CH * px * 2));
      if (use_color) c.rgb.reset((uint8_t*)scn_host_alloc(CH * px * 3));
      if (!c.depth || (use_color && !c.rgb)) fail.set(SCN_ERR_CUDA);
    }
    uint64_t f = 0; int cur = 0;
    if (!fail && in.n_frames) decode_chunk(s, in, lut, use_color, 0, (uint32_t)std::min<uint64_t>(CH, in.n_frames), ch[0], pool, fail);
    while (f < in.n_frames && !fail) {
      Chunk& c = ch[cur];
      // the GPU consumes chunk `cur` asynchronously while the host decodes the next one into the other buffer
      if (int r = scn_tsdf_integrate_batch(vol, c.n, c.depth.get(), c.rgb.get(), c.poses.data(), in.depth_intrinsic)) { fail.set(r); break; }
      f += c.n;
      if (f < in.n_frames) decode_chunk(s, in, lut, use_color, f, (uint32_t)std::min<uint64_t>(CH, in.n_frames - f), ch[cur ^ 1], pool, fail);
      if (int r = scn_tsdf_sync(vol)) { fail.set(r); break; }      // chunk `cur` may be overwritten next round
      cur ^= 1;
    }
  }
  if (gpu_decode) rep.teardown_s = now_s() - tt0;
  rep.fuse_s = now_s() - t0;
  if (!fail) {
    scn_tsdf_stats_t st; scn_tsdf_stats(vol, &st);
    rep.frames_integrated = st.frames_integrated; rep.frames_skipped = st.frames_skipped + rep.frames_skipped_pose;
    rep.blocks_allocated = st.blocks_allocated; rep.voxels_updated = st.voxels_updated;
    if (job.verbose)
      printf("integrated %llu frames (%llu skipped: invalid pose) in %.3f s = %.1f frames/s incl. decode; %llu blocks, %llu voxel updates\n",
             (unsigned long long)rep.frames_integrated, (unsigned long long)rep.frames_skipped, rep.fuse_s, rep.frames_integrated / std::max(rep.fuse_s, 1e-9),
             (unsigned long long)st.blocks_allocated, (unsigned long long)st.voxels_updated);
    size_t used = 0, total = 0;
    if (!scn_device_mem_info(&used, &total)) rep.device_bytes_in_use = used;
    if (!job.out_path.empty()) {
      const double tm0 = now_s();
      float* xyz = nullptr; uint8_t* rgb = nullptr; uint32_t* tri = nullptr; uint64_t nV = 0, nF = 0;
      if (int r = scn_tsdf_extract_mesh(vol, &xyz, &rgb, &tri, &nV, &nF)) fail.set(r);
      const scn::MallocPtr<float> own_xyz(xyz); const scn::MallocPtr<uint8_t> own_rgb(rgb); const scn::MallocPtr<uint32_t> own_tri(tri);
      rep.mc_s = now_s() - tm0;
      if (!fail) { if (int r = scn_mesh_save_ply(job.out_path.c_str(), xyz, use_color ? rgb : nullptr, nV, tri, nF)) fail.set(r); }
      rep.ply_s = now_s() - tm0 - rep.mc_s;
      rep.mesh_vertices = nV; rep.mesh_faces = nF;
      if (!fail && job.verbose) printf("mesh written to %s with %llu vertices, %llu faces\n", job.out_path.c_str(), (unsigned long long)nV, (unsigned long long)nF);
    }
  }
  if (fail) vs->release();                                     // do not hand a volume of unknown state to the next scene
  return fail ? scn::fail(fail.rc.load(), "%s: %s", job.sens_path.c_str(), fail.err.c_str()) : SCN_OK;
}

std::string default_out(const std::string& sens_path) { return sens_path.substr(0, sens_path.size() - 5) + "_vh.ply"; }

}  // namespace

int scn::fuse_sens(const scn_sens* s, const char* label, const char* out_ply, const scn_tsdf_params* params, int device, scn_fuse_report_t* report) {
  SceneJob j; j.sens_path = label; j.out_path = out_ply ? out_ply : ""; j.params = *params; j.device = device; j.verbose = false;
  scn_fuse_report_t rep; memset(&rep, 0, sizeof(rep));
  rep.device = device;
  const double t_begin = now_s();
  if (int r = scn_set_device(device)) return r;
  const int rc = fuse_open_scene(j, s, rep, t_begin);
  rep.total_s = now_s() - t_begin;
  if (report) *report = rep;
  return rc;
}

extern "C" {

void scn_fuse_release_staging_() { frame_pool().trim(); vol_pool().trim(); }
size_t scn_fuse_report_sizeof(void) { return sizeof(scn_fuse_report_t); }

int scn_fuse_scene(const char* sens_path, const char* out_ply, const scn_tsdf_params* params, int device, const char* decode_mode, scn_fuse_report_t* report) {
  if (!sens_path || !params) return scn::fail(SCN_ERR_ARG, "null argument");
  SceneJob j; j.sens_path = sens_path; j.out_path = out_ply ? out_ply : ""; j.params = *params; j.device = device; j.verbose = false; j.decode_mode = decode_mode;
  return fuse_scene(j, report);
}

// One scene per GPU at a time: worker d takes the next scene of the list, fuses it on devices[d], repeats.  No data-path
// collective (SURVEY.md §8e): the scenes are independent.
int scn_fuse_many(const char* const* sens_paths, const char* const* out_plys, uint32_t n_scenes, const scn_tsdf_params* params,
                  const int* devices, uint32_t n_devices, const char* decode_mode, scn_fuse_report_t* reports) {
  if (!sens_paths || !params || (!devices && n_devices) || !n_devices) return scn::fail(SCN_ERR_ARG, "null argument");
  std::atomic<uint32_t> next{0}; std::atomic<int> rc{0};
  std::mutex em; std::string first_err;
  auto worker = [&](int dev) {
    for (;;) {
      const uint32_t i = next.fetch_add(1);
      if (i >= n_scenes) break;
      SceneJob j; j.sens_path = sens_paths[i]; j.out_path = out_plys && out_plys[i] ? out_plys[i] : ""; j.params = *params; j.device = dev; j.verbose = false;
      j.decode_mode = decode_mode;
      scn_fuse_report_t r; memset(&r, 0, sizeof(r));
      const int e = fuse_scene(j, &r);
      r.status = e;
      if (reports) reports[i] = r;
      if (e) { std::lock_guard<std::mutex> l(em); if (!rc.load()) { first_err = scn_last_error(); rc.store(e); } }
    }
  };
  std::vector<std::thread> th;
  for (uint32_t d = 1; d < n_devices; ++d) th.emplace_back(worker, devices[d]);
  worker(devices[0]);
  for (auto& t : th) t.join();
  return rc.load() ? scn::fail(rc.load(), "%s", first_err.c_str()) : SCN_OK;
}

int scn_fuse_main(int argc, const char** argv) {
  std::vector<std::string> params, scenes; std::string out_path; int gpus = 0;
  for (int i = 1; i < argc; ++i) {
    const std::string a = argv[i];
    if (a == "--gpus" && i + 1 < argc) { gpus = atoi(argv[++i]); continue; }
    if (a.size() > 5 && a.substr(a.size() - 5) == ".sens") scenes.push_back(a);
    else if (!scenes.empty()) out_path = a;
    else params.push_back(a);
  }
  if (scenes.empty()) {
    printf("Usage: fuse <params.txt> [<params2.txt>] <file.sens> [out.ply]\n       fuse --gpus N <params.txt> ... <a.sens> <b.sens> ...\n");
    return 255;
  }
  scn_tsdf_params p; scn_tsdf_default_params(&p);
  p.max_blocks = 1ull << 22; p.hash_slots = 1ull << 24;      // 16 GiB of voxel blocks unless the parameter file says otherwise (s_hashNumSDFBlocks)
  for (const std::string& f : params) if (scn_tsdf_params_from_file(f.c_str(), &p)) { fprintf(stderr, "%s\n", scn_last_error()); return 1; }
  p.batch_frames = 32;
  const char* mode = getenv("SCN_FUSE_DECODE");
  if (scenes.size() == 1 && gpus <= 1) {
    SceneJob j; j.sens_path = scenes[0]; j.out_path = out_path.empty() ? default_out(scenes[0]) : out_path; j.params = p; j.device = 0; j.verbose = true; j.decode_mode = mode;
    scn_fuse_report_t r;
    if (fuse_scene(j, &r)) { fprintf(stderr, "%s\n", scn_last_error()); return 1; }
    if (getenv("SCN_TIMING"))
      fprintf(stderr, "[timing] fuse %.3f s (waiting for the decoders %.3f s; depth decode %.3f s, colour decode %.3f s on their threads), marching cubes %.3f s, PLY %.3f s, total %.3f s, %.2f GB of HBM in use\n",
              r.fuse_s, r.decode_wait_s, r.depth_decode_s, r.color_decode_s, r.mc_s, r.ply_s, r.total_s, r.device_bytes_in_use / 1e9);
    return 0;
  }
  int ndev = scn_device_count();
  if (ndev <= 0) { fprintf(stderr, "%s\n", scn_last_error()); return 1; }
  if (gpus <= 0 || gpus > ndev) gpus = ndev;
  gpus = std::min<int>(gpus, (int)scenes.size());
  std::vector<const char*> sp, op; std::vector<std::string> outs; std::vector<int> devs;
  for (const std::string& s : scenes) outs.push_back(default_out(s));
  for (size_t i = 0; i < scenes.size(); ++i) { sp.push_back(scenes[i].c_str()); op.push_back(outs[i].c_str()); }
  for (int d = 0; d < gpus; ++d) devs.push_back(d);
  std::vector<scn_fuse_report_t> reps(scenes.size());
  const double t0 = now_s();
  const int rc = scn_fuse_many(sp.data(), op.data(), (uint32_t)scenes.size(), &p, devs.data(), (uint32_t)devs.size(), mode, reps.data());
  const double dt = now_s() - t0;
  uint64_t frames = 0;
  for (size_t i = 0; i < scenes.size(); ++i) {
    const scn_fuse_report_t& r = reps[i];
    printf("%s: GPU %d, %llu frames in %.3f s = %.1f frames/s incl. decode, mesh %llu vertices / %llu faces%s\n", scenes[i].c_str(), r.device,
           (unsigned long long)r.frames_integrated, r.fuse_s, r.frames_integrated / std::max(r.fuse_s, 1e-9), (unsigned long long)r.mesh_vertices,
           (unsigned long long)r.mesh_faces, r.status ? "  FAILED" : "");
    frames += r.frames_integrated;
  }
  printf("%zu scenes on %d GPUs: %llu frames in %.3f s wall = %.1f frames/s aggregate (file -> TSDF -> mesh)\n", scenes.size(), gpus, (unsigned long long)frames, dt, frames / std::max(dt, 1e-9));
  if (rc) { fprintf(stderr, "%s\n", scn_last_error()); return 1; }
  return 0;
}

}  // extern "C"
