// Host side of the render stage (DESIGN.md §6i): the camera of Server/mts_render.py:69-106 in binary64, and `render`, the
// script's command line (the kernels and scn_render_mesh are in render.cu).
#include <cmath>
#include <algorithm>
#include <string>
#include <thread>
#include <vector>

#include "scn_common.h"

namespace scn {
void png_encode_stb(const uint8_t* px, uint32_t w, uint32_t h, int n, std::vector<uint8_t>& out);   // sens.cpp
}

namespace {

struct V3 { double x, y, z; };
V3 operator+(V3 a, V3 b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
V3 operator-(V3 a, V3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
V3 operator*(double s, V3 a) { return {s * a.x, s * a.y, s * a.z}; }
double dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
V3 cross(V3 a, V3 b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
double len(V3 a) { return std::sqrt(dot(a, a)); }
V3 v3(const float* f) { return {f[0], f[1], f[2]}; }

// Mitsuba's Transform::rotate(axis, angle in degrees): Rodrigues' matrix about the normalised axis
struct M3 { double m[3][3]; V3 operator*(V3 v) const { return {m[0][0] * v.x + m[0][1] * v.y + m[0][2] * v.z, m[1][0] * v.x + m[1][1] * v.y + m[1][2] * v.z,
                                                                  m[2][0] * v.x + m[2][1] * v.y + m[2][2] * v.z}; } };
M3 rotate(V3 axis, double deg) {
  const V3 a = (1.0 / len(axis)) * axis;
  const double rad = deg * (M_PI / 180.0), s = std::sin(rad), c = std::cos(rad), k = 1.0 - c;
  M3 r;
  r.m[0][0] = a.x * a.x + (1.0 - a.x * a.x) * c; r.m[0][1] = a.x * a.y * k - a.z * s;           r.m[0][2] = a.x * a.z * k + a.y * s;
  r.m[1][0] = a.x * a.y * k + a.z * s;           r.m[1][1] = a.y * a.y + (1.0 - a.y * a.y) * c; r.m[1][2] = a.y * a.z * k - a.x * s;
  r.m[2][0] = a.x * a.z * k - a.y * s;           r.m[2][1] = a.y * a.z * k + a.x * s;           r.m[2][2] = a.z * a.z + (1.0 - a.z * a.z) * c;
  return r;
}

bool finite3(const float* f) { return std::isfinite(f[0]) && std::isfinite(f[1]) && std::isfinite(f[2]); }

int write_file(const std::string& path, const std::vector<uint8_t>& bytes) {
  FILE* f = fopen(path.c_str(), "wb");
  if (!f) return scn::fail(SCN_ERR_IO, "cannot open %s for writing", path.c_str());
  const bool ok = fwrite(bytes.data(), 1, bytes.size(), f) == bytes.size();
  if (fclose(f) != 0 || !ok) return scn::fail(SCN_ERR_IO, "cannot write %s", path.c_str());
  return SCN_OK;
}

// mts_render.py's vec3 / nvec3: "x", "y", "z" or "a,b,c"; nvec3 normalises
bool parse_vec(const std::string& s, float out[3]) {
  double v[3] = {0, 0, 0};
  if (s == "x") v[0] = 1; else if (s == "y") v[1] = 1; else if (s == "z") v[2] = 1;
  else {
    size_t pos = 0;
    for (int i = 0; i < 3; ++i) {
      const size_t e = i < 2 ? s.find(',', pos) : s.size();
      if (e == std::string::npos) return false;
      const std::string t = s.substr(pos, e - pos);
      char* end = nullptr;
      v[i] = strtod(t.c_str(), &end);
      if (t.empty() || *end || !std::isfinite(v[i])) return false;
      pos = e + 1;
    }
  }
  const double l = std::sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
  if (!(l > 0)) return false;
  for (int i = 0; i < 3; ++i) out[i] = (float)(v[i] / l);
  return true;
}

bool parse_int(const std::string& s, int64_t& v) { char* e = nullptr; v = strtoll(s.c_str(), &e, 10); return !s.empty() && !*e; }
bool parse_num(const std::string& s, double& v) { char* e = nullptr; v = strtod(s.c_str(), &e); return !s.empty() && !*e && std::isfinite(v); }

}  // namespace

extern "C" {

int scn_render_camera(const float* xyz, uint64_t n_verts, const scn_render_params* p, double theta, int turntable, scn_render_camera_t* cam) {
  if (!xyz || !p || !cam) return scn::fail(SCN_ERR_ARG, "null argument");
  if (!n_verts) return scn::fail(SCN_ERR_ARG, "no vertex");
  if (p->width < 1 || p->height < 1) return scn::fail(SCN_ERR_ARG, "empty film %ux%u", p->width, p->height);
  if (!finite3(p->world_up) || !finite3(p->camera_up) || !finite3(p->camera_offset) || !std::isfinite(p->bsphere_mult) || !std::isfinite(theta))
    return scn::fail(SCN_ERR_ARG, "non-finite camera parameter");
  V3 lo = {INFINITY, INFINITY, INFINITY}, hi = {-INFINITY, -INFINITY, -INFINITY};
  for (uint64_t i = 0; i < n_verts; ++i) {
    const float* v = xyz + 3 * i;
    if (!finite3(v)) return scn::fail(SCN_ERR_ARG, "vertex %llu is not finite", (unsigned long long)i);
    lo = {std::min(lo.x, (double)v[0]), std::min(lo.y, (double)v[1]), std::min(lo.z, (double)v[2])};
    hi = {std::max(hi.x, (double)v[0]), std::max(hi.y, (double)v[1]), std::max(hi.z, (double)v[2])};
  }
  // mts_render.py:69-82: the AABB's bounding sphere, origin = c + bsphere_mult * r * normalize(camera_offset + world_up)
  const V3 c = 0.5 * (lo + hi);
  const double r = len(hi - c);
  const V3 up = v3(p->world_up), off = v3(p->camera_offset) + up;
  if (!(len(up) > 0) || !(len(off) > 0)) return scn::fail(SCN_ERR_ARG, "world_up and camera_offset + world_up must be non-zero");
  V3 origin = c + ((double)p->bsphere_mult * r / len(off)) * off;
  V3 cam_up = v3(p->camera_up);
  // :87-88 turntable: about the axis through c; :97-98 single view: about the world origin
  const M3 R = rotate(up, theta);
  origin = turntable ? c + R * (origin - c) : R * origin;
  cam_up = R * cam_up;
  // Transform::lookAt(origin, c, cam_up): dir, left = normalize(cross(up, dir)), newUp = cross(dir, left).  The film's x axis
  // runs along -left = cross(dir, up) and its y axis (down) along -newUp, so the image is not mirrored.
  const V3 fwd0 = c - origin;
  if (!(len(fwd0) > 0)) return scn::fail(SCN_ERR_ARG, "the camera sits at the target (radius %g, bsphere_mult %g)", r, (double)p->bsphere_mult);
  const V3 fwd = (1.0 / len(fwd0)) * fwd0;
  const V3 left0 = cross(cam_up, fwd);
  if (!(len(left0) > 1e-9 * len(cam_up))) return scn::fail(SCN_ERR_ARG, "camera_up is parallel to the view direction");
  const V3 left = (1.0 / len(left0)) * left0, new_up = cross(fwd, left);
  const double th = std::tan(22.5 * (M_PI / 180.0)), step = 2.0 * th / p->width;
  const V3 right = -1.0 * left;
  const V3 du = step * right, dv = -step * new_up;
  const V3 p00 = fwd - th * right + (th * p->height / p->width) * new_up;
  const V3* src[4] = {&origin, &p00, &du, &dv};
  float* dst[4] = {cam->origin, cam->p00, cam->du, cam->dv};
  for (int k = 0; k < 4; ++k) { dst[k][0] = (float)src[k]->x; dst[k][1] = (float)src[k]->y; dst[k][2] = (float)src[k]->z; }
  cam->t_near = 0.01f;
  cam->t_eps = (float)std::ldexp(r, -16);
  cam->ao_length = (float)r;
  return SCN_OK;
}

int scn_render_main(int argc, const char** argv) {
  scn_render_params p; scn_render_default_params(&p);
  std::string out, mesh;
  double theta = 0;
  int64_t fpd = 5;
  bool turntable = false;
  auto usage = [](const char* why) {
    fprintf(stderr, "render: %s\nUsage: render [-o out.png] [--integrator path|ao] [--samples N] [--width W] [--height H] [--theta T]\n"
                    "              [--exposure E] [--world_up v] [--camera_up v] [--camera_offset v] [--bsphere_mult M]\n"
                    "              [--render_turntable] [--frames_per_degree D] mesh.ply\n", why);
    return 2;
  };
  for (int i = 1; i < argc; ++i) {
    std::string a = argv[i], val;
    bool has_val = false;
    const size_t eq = a.rfind("--", 0) == 0 ? a.find('=') : std::string::npos;
    if (eq != std::string::npos) { val = a.substr(eq + 1); a = a.substr(0, eq); has_val = true; }
    else if (a.size() > 2 && a.rfind("-o", 0) == 0) { val = a.substr(2); a = "-o"; has_val = true; }
    if (a == "--render_turntable") { if (has_val) return usage("--render_turntable takes no value"); turntable = true; continue; }
    if (a == "--cameras") { scn::fail(SCN_ERR_UNSUPPORTED, "--cameras is not supported (mts_render.py parses it but never reads it)");
                            fprintf(stderr, "render: %s\n", scn_last_error()); return 1; }
    if (a.size() > 1 && a[0] == '-' && a != "-") {
      if (!has_val) { if (i + 1 >= argc) return usage(("missing value for " + a).c_str()); val = argv[++i]; }
      double d = 0; int64_t n = 0;
      if (a == "-o") out = val;
      else if (a == "--integrator") {
        if (val == "path") p.integrator = SCN_RENDER_PATH;
        else if (val == "ao") p.integrator = SCN_RENDER_AO;
        else if (val == "mlt" || val == "vpl") { scn::fail(SCN_ERR_UNSUPPORTED, "integrator '%s' is not supported (path and ao are)", val.c_str());
                                                 fprintf(stderr, "render: %s\n", scn_last_error()); return 1; }
        else return usage(("invalid integrator '" + val + "' (choose from path, mlt, vpl, ao)").c_str());
      }
      else if (a == "--samples" && parse_int(val, n) && n >= 1 && n <= UINT32_MAX) p.samples = (uint32_t)n;
      else if (a == "--width" && parse_int(val, n) && n >= 1 && n <= UINT32_MAX) p.width = (uint32_t)n;
      else if (a == "--height" && parse_int(val, n) && n >= 1 && n <= UINT32_MAX) p.height = (uint32_t)n;
      else if (a == "--frames_per_degree" && parse_int(val, n) && n >= 1 && n <= 360) fpd = n;
      else if (a == "--theta" && parse_num(val, d)) theta = d;
      else if (a == "--exposure" && parse_num(val, d)) p.exposure = (float)d;
      else if (a == "--bsphere_mult" && parse_num(val, d)) p.bsphere_mult = (float)d;
      else if (a == "--world_up" && parse_vec(val, p.world_up)) {}
      else if (a == "--camera_up" && parse_vec(val, p.camera_up)) {}
      else if (a == "--camera_offset" && parse_vec(val, p.camera_offset)) {}
      else return usage(("invalid argument " + a + " " + val).c_str());
      continue;
    }
    if (!mesh.empty()) return usage(("unrecognised argument " + a).c_str());
    mesh = a;
  }
  if (mesh.empty()) return usage("the mesh argument is required");
  const double t0 = scn::now_s();
  float* x = nullptr; uint8_t* rgb = nullptr; uint32_t* t = nullptr; uint64_t nv = 0, nf = 0;
  const int lrc = scn_mesh_load_rgb(mesh.c_str(), &x, &rgb, &nv, &t, &nf);
  scn::MallocPtr<float> hx(x); scn::MallocPtr<uint8_t> hc(rgb); scn::MallocPtr<uint32_t> ht(t);
  if (lrc) { fprintf(stderr, "render: %s\n", scn_last_error()); return 1; }
  // one view, or floor(360 / D) turntable frames D degrees apart ('{0}_%03i.png'.format(meshfile) % i, mts_render.py:83-92)
  const uint32_t n_views = turntable ? (uint32_t)(360 / fpd) : 1;
  std::vector<scn_render_camera_t> cams(n_views);
  std::vector<std::string> names(n_views);
  for (uint32_t i = 0; i < n_views; ++i) {
    const int rc = scn_render_camera(x, nv, &p, turntable ? (double)(i * fpd) : theta, turntable, &cams[i]);
    if (rc) { fprintf(stderr, "render: %s\n", scn_last_error()); return 1; }
    if (turntable) { char b[16]; snprintf(b, sizeof(b), "_%03u.png", i); names[i] = mesh + b; }
  }
  if (!turntable) {
    if (!out.empty()) names[0] = out;
    else {
      // os.path.splitext: the extension starts at the last dot of the last component, unless that component starts with it
      const size_t slash = mesh.rfind('/'), base = slash == std::string::npos ? 0 : slash + 1;
      size_t dot = mesh.rfind('.');
      size_t b = base; while (b < mesh.size() && mesh[b] == '.') ++b;
      if (dot == std::string::npos || dot < b) dot = mesh.size();
      names[0] = mesh.substr(0, dot) + ".png";
    }
  }
  const size_t frame = (size_t)p.width * p.height * 4;
  std::vector<uint8_t> rgba(frame * n_views);
  scn_render_report_t rep;
  if (scn_render_mesh(x, rgb, nv, t, nf, &p, cams.data(), n_views, rgba.data(), &rep)) { fprintf(stderr, "render: %s\n", scn_last_error()); return 1; }
  // the frames are encoded and written on up to 16 threads (a turntable is 72 PNGs); the first failure is reported
  const double t_png = scn::now_s();
  const uint32_t n_thr = std::min<uint32_t>(n_views, std::max(1u, std::min(16u, std::thread::hardware_concurrency())));
  std::vector<int> rcs(n_views, SCN_OK);
  std::vector<std::string> errs(n_views);
  std::vector<std::thread> pool;
  for (uint32_t k = 0; k < n_thr; ++k)
    pool.emplace_back([&, k]() {
      std::vector<uint8_t> png;
      for (uint32_t i = k; i < n_views; i += n_thr) {
        scn::png_encode_stb(rgba.data() + frame * i, p.width, p.height, 4, png);
        if ((rcs[i] = write_file(names[i], png))) errs[i] = scn_last_error();
      }
    });
  for (auto& th : pool) th.join();
  for (uint32_t i = 0; i < n_views; ++i)
    if (rcs[i]) { fprintf(stderr, "render: %s\n", errs[i].c_str()); return 1; }
  const double png_ms = (scn::now_s() - t_png) * 1e3;
  printf("render %s: %llu faces, %u view(s) %ux%u at %u spp (%s): %llu primary + %llu secondary rays, bvh %.1f ms, trace %.1f ms, "
         "png %.1f ms; %.3f s -> %s%s\n",
         mesh.c_str(), (unsigned long long)nf, n_views, p.width, p.height, p.samples, p.integrator == SCN_RENDER_AO ? "ao" : "path",
         (unsigned long long)rep.primary_rays, (unsigned long long)rep.secondary_rays, rep.bvh_ms, rep.trace_ms, png_ms, scn::now_s() - t0, names[0].c_str(),
         n_views > 1 ? " ..." : "");
  return 0;
}

}  // extern "C"
