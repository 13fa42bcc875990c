// Mesh I/O + the Segmentator command line, host side (C++).
//
//   scn_mesh_load          the two loaders of segment() (/root/reference/Segmentator/segmentator.cpp:130-172):
//       .ply  tinyply semantics as the reference uses them (tinyply.h:222-313, tinyply.cpp:62-360): header-driven,
//             ascii / binary little / big endian, vertex x,y,z as 4-byte floats, faces from the list property
//             "vertex_indices" (or "vertex_index") with 4-byte indices, three per face; everything else skipped.
//       .obj  tinyobjloader semantics as the reference uses them (LoadObj(..., triangulate=false), first shape
//             only, original vertices kept): including its hand-rolled decimal parser (tiny_obj_loader.h:505-618),
//             whose results can differ from strtod in the last ulp and therefore decide float bit patterns.
//   scn_write_segs_json    writeToJSON (segmentator.cpp:253-266)
//   scn_segmentator_main   main (segmentator.cpp:268-288): same argv, stdout lines, file naming, exit codes
//   scn_mesh_save_ply      VCGLIB-layout binary PLY (the layout of gates381.ply / ScanNet *_vh_clean*.ply)
#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <iostream>
#include <sstream>
#include <string>
#include <thread>
#include <unordered_set>
#include <vector>

#include "scn_common.h"

namespace {

bool ends_with(const std::string& v, const std::string& e) { return e.size() <= v.size() && std::equal(e.rbegin(), e.rend(), v.rbegin()); }

// ------------------------------------------------------------------------------ PLY
enum PType { T_I8, T_U8, T_I16, T_U16, T_I32, T_U32, T_F32, T_F64, T_BAD };
int psize(PType t) { static const int s[] = {1, 1, 2, 2, 4, 4, 4, 8, 0}; return s[t]; }
PType ptype(const std::string& t) {
  if (t == "int8" || t == "char") return T_I8; if (t == "uint8" || t == "uchar") return T_U8;
  if (t == "int16" || t == "short") return T_I16; if (t == "uint16" || t == "ushort") return T_U16;
  if (t == "int32" || t == "int") return T_I32; if (t == "uint32" || t == "uint") return T_U32;
  if (t == "float32" || t == "float") return T_F32; if (t == "float64" || t == "double") return T_F64;
  return T_BAD;
}
struct PProp { std::string name; PType type = T_BAD, list_type = T_BAD; bool is_list = false; };
struct PElem { std::string name; size_t count = 0; std::vector<PProp> props; };

inline uint64_t load_le(const uint8_t* p, int n, bool big) {
  uint64_t v = 0;
  if (big) for (int i = 0; i < n; ++i) v = (v << 8) | p[i]; else for (int i = n - 1; i >= 0; --i) v = (v << 8) | p[i];
  return v;
}
inline int64_t as_int(const uint8_t* p, PType t, bool big) {
  const uint64_t u = load_le(p, psize(t), big);
  switch (t) { case T_I8: return (int8_t)u; case T_U8: return (uint8_t)u; case T_I16: return (int16_t)u; case T_U16: return (uint16_t)u;
    case T_I32: return (int32_t)u; case T_U32: return (uint32_t)u; default: return 0; }
}

// rgb != nullptr: also the vertex colour when the vertex element has uchar red, green and blue (else rgb stays empty)
int load_ply(const std::string& path, std::vector<float>& xyz, std::vector<uint32_t>& tri, std::vector<uint8_t>* rgb = nullptr) {
  // the file is mapped, not read: a 2 M-vertex mesh is 84 MB and the arrays below are the only copy that is needed
  struct FileView {
    const uint8_t* p = nullptr; size_t n = 0; bool mapped = false; std::vector<uint8_t> own;
    ~FileView() { if (mapped) munmap(const_cast<uint8_t*>(p), n); }
    const uint8_t* data() const { return p; }
    size_t size() const { return n; }
    uint8_t operator[](size_t i) const { return p[i]; }
  } buf;
  {
    const int fd = ::open(path.c_str(), O_RDONLY);
    if (fd < 0) return scn::fail(SCN_ERR_IO, "cannot open %s", path.c_str());
    struct stat st;
    if (fstat(fd, &st) != 0 || S_ISDIR(st.st_mode)) { ::close(fd); return scn::fail(SCN_ERR_IO, "cannot open %s", path.c_str()); }
    const size_t fsz = (size_t)std::max<off_t>(st.st_size, 0);
    if (fsz) {
      void* m = mmap(nullptr, fsz, PROT_READ, MAP_PRIVATE | MAP_POPULATE, fd, 0);
      if (m != MAP_FAILED) { buf.p = (const uint8_t*)m; buf.n = fsz; buf.mapped = true; }
      else {
        buf.own.resize(fsz);
        size_t got = 0;
        while (got < fsz) { const ssize_t r = ::read(fd, buf.own.data() + got, fsz - got); if (r <= 0) break; got += (size_t)r; }
        if (got != fsz) { ::close(fd); return scn::fail(SCN_ERR_IO, "short read on %s", path.c_str()); }
        buf.p = buf.own.data(); buf.n = fsz;
      }
    }
    ::close(fd);
  }
  // header
  size_t pos = 0; bool binary = false, big = false, done = false; std::vector<PElem> elems;
  while (pos < buf.size() && !done) {
    size_t e = pos; while (e < buf.size() && buf[e] != '\n') ++e;
    std::string line((const char*)buf.data() + pos, e - pos); pos = e + 1;
    std::istringstream ls(line); std::string tok; ls >> tok;
    if (tok == "ply" || tok == "PLY" || tok == "") continue;
    else if (tok == "comment" || tok == "obj_info") continue;
    else if (tok == "format") { std::string s; ls >> s; if (s == "binary_little_endian") binary = true; else if (s == "binary_big_endian") binary = big = true; }
    else if (tok == "element") { PElem el; ls >> el.name >> el.count; elems.push_back(el); }
    else if (tok == "property") {
      if (elems.empty()) return scn::fail(SCN_ERR_FORMAT, "file is not ply or encounted junk in header");
      PProp p; std::string t; ls >> t;
      if (t == "list") { std::string ct; ls >> ct >> t; p.list_type = ptype(ct); p.is_list = true; }
      p.type = ptype(t); ls >> p.name; elems.back().props.push_back(p);
    } else if (tok == "end_header") done = true;
    else return scn::fail(SCN_ERR_FORMAT, "file is not ply or encounted junk in header");   // tinyply.cpp:58
  }
  if (!done) return scn::fail(SCN_ERR_FORMAT, "PLY header has no end_header");
  // which face list property (segmentator.cpp:136-139)
  std::string face_prop;
  for (const PElem& el : elems) if (el.name == "face") {
    for (const PProp& p : el.props) if (p.name == "vertex_indices") face_prop = p.name;
    if (face_prop.empty()) for (const PProp& p : el.props) if (p.name == "vertex_index") face_prop = p.name;
  }
  bool have_xyz = false;
  for (const PElem& el : elems) if (el.name == "vertex") {
    int got = 0;
    for (const PProp& p : el.props) if (!p.is_list && (p.name == "x" || p.name == "y" || p.name == "z")) {
      if (psize(p.type) != 4) return scn::fail(SCN_ERR_FORMAT, "destination vector is wrongly typed to hold this property");   // tinyply.h:245-246
      if (p.type != T_F32) return scn::fail(SCN_ERR_UNSUPPORTED, "vertex property %s must be float32", p.name.c_str());
      ++got;
    }
    have_xyz = got == 3;
  }
  xyz.clear(); tri.clear();
  bool want_rgb = false;
  auto rgb_slot = [](const std::string& n) { return n == "red" ? 0 : n == "green" ? 1 : n == "blue" ? 2 : -1; };
  if (rgb) {
    rgb->clear();
    for (const PElem& el : elems) if (el.name == "vertex") {
      int got = 0;
      for (const PProp& p : el.props) if (!p.is_list && p.type == T_U8 && rgb_slot(p.name) >= 0) ++got;
      want_rgb = got == 3 && have_xyz;
    }
  }
  const uint8_t* d = buf.data(); const size_t n = buf.size();
  if (binary) {
    for (const PElem& el : elems) {
      const bool is_v = el.name == "vertex" && have_xyz, is_f = el.name == "face" && !face_prop.empty();
      // fast path: fixed-size records
      bool fixed = true; size_t rec = 0;
      for (const PProp& p : el.props) { if (p.is_list) fixed = false; rec += psize(p.type); if (p.type == T_BAD) return scn::fail(SCN_ERR_FORMAT, "invalid ply property"); }
      // bound the header's count by what the file can hold before any resize (overflow-safe: divide, never multiply)
      size_t min_rec = 0;
      for (const PProp& p : el.props) min_rec += p.is_list ? psize(p.list_type) : psize(p.type);
      if (el.count > (n - std::min(pos, n)) / std::max<size_t>(min_rec, 1)) return scn::fail(SCN_ERR_FORMAT, "PLY body truncated");
      if (is_v) xyz.resize(el.count * 3);
      if (is_v && want_rgb) rgb->resize(el.count * 3);
      if (is_f) tri.reserve(el.count * 3);
      if (fixed) {
        if (rec * el.count > n - pos) return scn::fail(SCN_ERR_FORMAT, "PLY body truncated");
        if (is_v) {
          size_t ox = 0, oy = 0, oz = 0, o = 0;
          for (const PProp& p : el.props) { if (p.name == "x") ox = o; else if (p.name == "y") oy = o; else if (p.name == "z") oz = o; o += psize(p.type); }
          if (!big && oy == ox + 4 && oz == ox + 8) {                 // x, y, z adjacent little-endian floats: 12 bytes per vertex
            const uint8_t* r = d + pos + ox;
            for (size_t i = 0; i < el.count; ++i, r += rec) memcpy(&xyz[3 * i], r, 12);
          } else for (size_t i = 0; i < el.count; ++i) {
            const uint8_t* r = d + pos + i * rec;
            uint32_t a = (uint32_t)load_le(r + ox, 4, big), b = (uint32_t)load_le(r + oy, 4, big), c = (uint32_t)load_le(r + oz, 4, big);
            memcpy(&xyz[3 * i], &a, 4); memcpy(&xyz[3 * i + 1], &b, 4); memcpy(&xyz[3 * i + 2], &c, 4);
          }
          if (want_rgb) {
            size_t oc[3] = {0, 0, 0}; o = 0;
            for (const PProp& p : el.props) { const int k = rgb_slot(p.name); if (k >= 0 && p.type == T_U8) oc[k] = o; o += psize(p.type); }
            for (size_t i = 0; i < el.count; ++i) for (int k = 0; k < 3; ++k) (*rgb)[3 * i + k] = d[pos + i * rec + oc[k]];
          }
        }
        pos += rec * el.count;
      } else if (is_f && el.props.size() == 1 && el.props[0].is_list && psize(el.props[0].list_type) == 1 && psize(el.props[0].type) == 4 &&
                 pos + 13 * el.count <= n && !big) {
        // the VCGLIB / ScanNet layout: `list uchar int vertex_indices`, 13-byte records when every face is a triangle
        bool all3 = true;
        for (size_t i = 0; i < el.count; ++i) if (d[pos + 13 * i] != 3) { all3 = false; break; }
        if (all3) {
          tri.resize(el.count * 3);
          for (size_t i = 0; i < el.count; ++i) memcpy(&tri[3 * i], d + pos + 13 * i + 1, 12);
          pos += 13 * el.count;
        } else return scn::fail(SCN_ERR_UNSUPPORTED, "only triangle meshes are supported (segmentator.cpp:136)");
      } else {
        for (size_t i = 0; i < el.count; ++i) {
          for (const PProp& p : el.props) {
            if (!p.is_list) {
              if (pos + psize(p.type) > n) return scn::fail(SCN_ERR_FORMAT, "PLY body truncated");
              if (is_v && (p.name == "x" || p.name == "y" || p.name == "z")) { uint32_t a = (uint32_t)load_le(d + pos, 4, big); memcpy(&xyz[3 * i + (p.name[0] - 'x')], &a, 4); }
              if (is_v && want_rgb && p.type == T_U8 && rgb_slot(p.name) >= 0) (*rgb)[3 * i + rgb_slot(p.name)] = d[pos];
              pos += psize(p.type);
            } else {
              if (p.list_type == T_BAD || p.list_type == T_F32 || p.list_type == T_F64) return scn::fail(SCN_ERR_FORMAT, "invalid ply list count type");
              if (pos + psize(p.list_type) > n) return scn::fail(SCN_ERR_FORMAT, "PLY body truncated");
              const int64_t cnt = as_int(d + pos, p.list_type, big); pos += psize(p.list_type);
              if (cnt < 0 || pos + (size_t)cnt * psize(p.type) > n) return scn::fail(SCN_ERR_FORMAT, "PLY body truncated");
              if (is_f && p.name == face_prop) {
                if (psize(p.type) != 4) return scn::fail(SCN_ERR_FORMAT, "destination vector is wrongly typed to hold this property");
                if (cnt != 3) return scn::fail(SCN_ERR_UNSUPPORTED, "face %zu has %lld vertices; only triangle meshes are supported (segmentator.cpp:136)", i, (long long)cnt);
                for (int k = 0; k < 3; ++k) tri.push_back((uint32_t)load_le(d + pos + 4 * k, 4, big));
              }
              pos += (size_t)cnt * psize(p.type);
            }
          }
        }
      }
    }
  } else {
    std::string body((const char*)d + pos, n - pos);
    std::istringstream is(body);
    for (const PElem& el : elems) {
      const bool is_v = el.name == "vertex" && have_xyz, is_f = el.name == "face" && !face_prop.empty();
      if (el.count > n - std::min(pos, n)) return scn::fail(SCN_ERR_FORMAT, "PLY body truncated");   // >= 1 byte per record
      if (is_v) xyz.resize(el.count * 3);
      if (is_v && want_rgb) rgb->resize(el.count * 3);
      for (size_t i = 0; i < el.count; ++i) for (const PProp& p : el.props) {
        if (!p.is_list) {
          if (is_v && (p.name == "x" || p.name == "y" || p.name == "z")) { float v = 0; is >> v; xyz[3 * i + (p.name[0] - 'x')] = v; }   // ply_cast_ascii<float>
          else if (is_v && want_rgb && p.type == T_U8 && rgb_slot(p.name) >= 0) { int v = 0; is >> v; (*rgb)[3 * i + rgb_slot(p.name)] = (uint8_t)v; }
          else { std::string s; is >> s; }
        } else {
          long long cnt = 0; is >> cnt;
          if (is_f && p.name == face_prop) {
            if (cnt != 3) return scn::fail(SCN_ERR_UNSUPPORTED, "face %zu has %lld vertices; only triangle meshes are supported", i, cnt);
            for (int k = 0; k < 3; ++k) { long long v = 0; is >> v; tri.push_back((uint32_t)v); }
          } else for (long long k = 0; k < cnt; ++k) { std::string s; is >> s; }
        }
        if (!is) return scn::fail(SCN_ERR_FORMAT, "PLY body truncated");
      }
    }
  }
  return SCN_OK;
}

// ------------------------------------------------------------------------------ OBJ
inline bool is_digit(char c) { return (unsigned)(c - '0') < 10u; }
bool obj_parse_double(const char* s, const char* s_end, double* result) {      // tiny_obj_loader.h:505-618
  if (s >= s_end) return false;
  double mantissa = 0.0; int exponent = 0; char sign = '+', exp_sign = '+'; const char* c = s; int read = 0; bool more = false;
  if (*c == '+' || *c == '-') { sign = *c; c++; } else if (!is_digit(*c)) return false;
  more = (c != s_end);
  while (more && is_digit(*c)) { mantissa *= 10; mantissa += (int)(*c - 0x30); c++; read++; more = (c != s_end); }
  if (read == 0) return false;
  if (more) {
    bool to_assemble = false;
    if (*c == '.') {
      c++; read = 1; more = (c != s_end);
      while (more && is_digit(*c)) {
        static const double lut[] = {1.0, 0.1, 0.01, 0.001, 0.0001, 0.00001, 0.000001, 0.0000001};
        mantissa += (int)(*c - 0x30) * (read < 8 ? lut[read] : std::pow(10.0, -read));
        read++; c++; more = (c != s_end);
      }
    } else if (*c == 'e' || *c == 'E') {
    } else to_assemble = true;
    if (!to_assemble && more && (*c == 'e' || *c == 'E')) {
      c++; more = (c != s_end);
      if (more && (*c == '+' || *c == '-')) { exp_sign = *c; c++; } else if (is_digit(*c)) {} else return false;
      read = 0; more = (c != s_end);
      while (more && is_digit(*c)) { exponent *= 10; exponent += (int)(*c - 0x30); c++; read++; more = (c != s_end); }
      exponent *= (exp_sign == '+' ? 1 : -1);
      if (read == 0) return false;
    }
  }
  *result = (sign == '+' ? 1 : -1) * (exponent ? std::ldexp(mantissa * std::pow(5.0, exponent), exponent) : mantissa);
  return true;
}
float obj_parse_real(const char** tok, double dflt = 0.0) {
  (*tok) += strspn(*tok, " \t");
  const char* end = (*tok) + strcspn(*tok, " \t\r");
  double v = dflt; obj_parse_double(*tok, end, &v);
  *tok = end;
  return (float)v;
}

int load_obj(const std::string& path, std::vector<float>& xyz, std::vector<uint32_t>& tri) {
  std::ifstream in(path, std::ios::binary);
  if (!in) return scn::fail(SCN_ERR_IO, "Cannot open file [%s]", path.c_str());
  std::string all((std::istreambuf_iterator<char>(in)), std::istreambuf_iterator<char>());
  xyz.clear(); tri.clear();
  std::vector<int> first_shape, cur;          // flattened vertex indices (triangulate = false keeps polygons as they are)
  size_t first_faces = 0, cur_faces = 0; bool have_first = false;
  auto flush = [&]() { if (!have_first && !cur.empty()) { first_shape.swap(cur); first_faces = cur_faces; have_first = true; } cur.clear(); cur_faces = 0; };
  size_t p = 0; const size_t n = all.size();
  while (p < n) {
    size_t e = p; while (e < n && all[e] != '\n' && all[e] != '\r') ++e;
    std::string line = all.substr(p, e - p);
    if (e < n && all[e] == '\r' && e + 1 < n && all[e + 1] == '\n') p = e + 2; else p = e + 1;     // safeGetline
    const char* t = line.c_str(); t += strspn(t, " \t");
    if (t[0] == '\0' || t[0] == '#') continue;
    auto sp = [](char c) { return c == ' ' || c == '\t'; };
    if (t[0] == 'v' && sp(t[1])) { t += 2; const float x = obj_parse_real(&t), y = obj_parse_real(&t), z = obj_parse_real(&t); xyz.push_back(x); xyz.push_back(y); xyz.push_back(z); continue; }
    if (t[0] == 'f' && sp(t[1])) {
      t += 2; t += strspn(t, " \t");
      while (!(t[0] == '\r' || t[0] == '\n' || t[0] == '\0')) {
        const int idx = atoi(t), nv = (int)(xyz.size() / 3);
        int v;
        if (idx > 0) v = idx - 1; else if (idx < 0) v = nv + idx;
        else return scn::fail(SCN_ERR_FORMAT, "Failed parse `f' line(e.g. zero value for face index).");
        cur.push_back(v);
        t += strcspn(t, "/ \t\r");
        while (t[0] == '/') { ++t; t += strcspn(t, "/ \t\r"); }        // vt / vn parts are irrelevant here
        t += strspn(t, " \t\r");
      }
      ++cur_faces;
      continue;
    }
    if ((t[0] == 'g' || t[0] == 'o') && sp(t[1])) { flush(); continue; }
  }
  flush();
  if (!have_first) return scn::fail(SCN_ERR_FORMAT, "OBJ file has no faces");
  if (first_shape.size() < 3 * first_faces) return scn::fail(SCN_ERR_UNSUPPORTED, "OBJ faces with fewer than 3 vertices");
  tri.resize(3 * first_faces);                                           // segmentator.cpp:163-170: 3 consecutive indices per face
  for (size_t i = 0; i < 3 * first_faces; ++i) tri[i] = (uint32_t)first_shape[i];
  return SCN_OK;
}


// ------------------------------------------------------------------------------ segs.json reader
// Minimal JSON walker: enough to read what Segmentator (and the annotation tools' re-savers) write, with the
// value tolerance of Segmentation::getUINT / getFloat (Segmentation.h:158-190).
struct JsonCur {
  const char* p; const char* e; std::string err;
  void ws() { while (p < e && (*p == ' ' || *p == '\n' || *p == '\r' || *p == '\t')) ++p; }
  bool eat(char c) { ws(); if (p < e && *p == c) { ++p; return true; } return false; }
  bool str(std::string& out) {
    ws(); if (p >= e || *p != '"') return false; ++p; out.clear();
    while (p < e && *p != '"') {
      if (*p == '\\' && p + 1 < e) { ++p; switch (*p) { case 'n': out.push_back('\n'); break; case 't': out.push_back('\t'); break; case 'r': out.push_back('\r'); break;
        case 'b': out.push_back('\b'); break; case 'f': out.push_back('\f'); break; case 'u': out.push_back('?'); p += (e - p > 4 ? 4 : 0); break; default: out.push_back(*p); } ++p; }
      else out.push_back(*p++);
    }
    if (p >= e) return false; ++p; return true;
  }
  bool skip() {                                                            // any value
    ws(); if (p >= e) return false;
    if (*p == '"') { std::string t; return str(t); }
    if (*p == '{' || *p == '[') {
      const char open = *p, close = open == '{' ? '}' : ']'; ++p;
      if (eat(close)) return true;
      for (;;) {
        if (open == '{') { std::string k; if (!str(k) || !eat(':')) return false; }
        if (!skip()) return false;
        if (eat(',')) continue;
        return eat(close);
      }
    }
    while (p < e && *p != ',' && *p != '}' && *p != ']' && *p != ' ' && *p != '\n' && *p != '\r' && *p != '\t') ++p;   // number / true / false / null
    return true;
  }
  // number | "digits" | null  ->  double (null: nan)
  bool num(double& v) {
    ws(); if (p >= e) return false;
    if (*p == '"') { std::string t; if (!str(t)) return false; v = atof(t.c_str()); return true; }
    if (e - p >= 4 && !strncmp(p, "null", 4)) { p += 4; v = NAN; return true; }
    char* end = nullptr; v = strtod(p, &end); if (end == p) return false; p = end; return true;
  }
};

}  // namespace

extern "C" {

int scn_mesh_load(const char* path, float** xyz, uint64_t* n_verts, uint32_t** tri, uint64_t* n_faces) {
  if (!path || !xyz || !n_verts || !tri || !n_faces) return scn::fail(SCN_ERR_ARG, "null argument");
  const std::string p = path;
  std::vector<float> v; std::vector<uint32_t> t;
  int rc;
  try {                                                                  // nothing crosses the C boundary as an exception
    if (ends_with(p, ".ply") || ends_with(p, ".PLY")) rc = load_ply(p, v, t);
    else if (ends_with(p, ".obj") || ends_with(p, ".OBJ")) rc = load_obj(p, v, t);
    else { v.clear(); t.clear(); rc = SCN_OK; }                          // segmentator.cpp:130,141: neither branch -> empty mesh
  } catch (const std::bad_alloc&) { return scn::fail(SCN_ERR_FORMAT, "mesh file %s: out of memory while parsing", path);
  } catch (const std::exception& e) { return scn::fail(SCN_ERR_FORMAT, "mesh file %s: %s", path, e.what()); }
  if (rc) return rc;
  *n_verts = v.size() / 3; *n_faces = t.size() / 3;
  *xyz = (float*)malloc(std::max<size_t>(1, v.size() * 4)); *tri = (uint32_t*)malloc(std::max<size_t>(1, t.size() * 4));
  if (!*xyz || !*tri) return scn::fail(SCN_ERR_ARG, "out of memory");
  memcpy(*xyz, v.data(), v.size() * 4); memcpy(*tri, t.data(), t.size() * 4);
  return SCN_OK;
}

int scn_mesh_load_rgb(const char* path, float** xyz, uint8_t** rgb, uint64_t* n_verts, uint32_t** tri, uint64_t* n_faces) {
  if (!path || !xyz || !rgb || !n_verts || !tri || !n_faces) return scn::fail(SCN_ERR_ARG, "null argument");
  *xyz = nullptr; *rgb = nullptr; *tri = nullptr; *n_verts = 0; *n_faces = 0;
  const std::string p = path;
  std::vector<float> v; std::vector<uint32_t> t; std::vector<uint8_t> c;
  int rc;
  try {
    if (ends_with(p, ".ply") || ends_with(p, ".PLY")) rc = load_ply(p, v, t, &c);
    else if (ends_with(p, ".obj") || ends_with(p, ".OBJ")) rc = load_obj(p, v, t);
    else rc = SCN_OK;
  } catch (const std::bad_alloc&) { return scn::fail(SCN_ERR_FORMAT, "mesh file %s: out of memory while parsing", path);
  } catch (const std::exception& e) { return scn::fail(SCN_ERR_FORMAT, "mesh file %s: %s", path, e.what()); }
  if (rc) return rc;
  *n_verts = v.size() / 3; *n_faces = t.size() / 3;
  *xyz = (float*)malloc(std::max<size_t>(1, v.size() * 4)); *tri = (uint32_t*)malloc(std::max<size_t>(1, t.size() * 4));
  if (!c.empty()) *rgb = (uint8_t*)malloc(c.size());
  if (!*xyz || !*tri || (!c.empty() && !*rgb)) return scn::fail(SCN_ERR_ARG, "out of memory");
  memcpy(*xyz, v.data(), v.size() * 4); memcpy(*tri, t.data(), t.size() * 4);
  if (!c.empty()) memcpy(*rgb, c.data(), c.size());
  return SCN_OK;
}

int scn_write_segs_json(const char* path, const char* scene_id, float k_thresh, int32_t seg_min_verts, const int32_t* seg, uint64_t n) {
  if (!path || !scene_id || (!seg && n)) return scn::fail(SCN_ERR_ARG, "null argument");
  std::ostringstream hd;                                                // same stream formatting as the reference's ofstream
  hd << "{";
  hd << "\"params\":{\"kThresh\":" << k_thresh << ",\"segMinVerts\":" << seg_min_verts << "},";
  hd << "\"sceneId\":\"" << scene_id << "\",";
  hd << "\"segIndices\":[";
  std::string body = hd.str();
  // "%d" of every id, comma separated (2 M ids took 0.14 s through snprintf; this loop writes the digits directly)
  const size_t head = body.size();
  body.resize(head + n * 12 + 8);
  char* w = &body[head];
  for (uint64_t i = 0; i < n; ++i) {
    if (i > 0) *w++ = ',';
    int64_t v = seg[i];
    if (v < 0) { *w++ = '-'; v = -v; }
    char tmp[12]; int k = 0;
    do { tmp[k++] = (char)('0' + v % 10); v /= 10; } while (v);
    while (k) *w++ = tmp[--k];
  }
  *w++ = ']'; *w++ = '}';
  body.resize((size_t)(w - body.data()));
  FILE* f = fopen(path, "wb");
  if (!f) return scn::fail(SCN_ERR_IO, "cannot write %s", path);
  const bool ok = fwrite(body.data(), 1, body.size(), f) == body.size();
  fclose(f);
  return ok ? SCN_OK : scn::fail(SCN_ERR_IO, "short write on %s", path);
}

int scn_segs_load(const char* path, uint32_t** seg_out, uint64_t* n_out, float* k_thresh, uint32_t* seg_min_verts, char* scene_id, size_t scene_id_cap) {
  if (!path || !seg_out || !n_out) return scn::fail(SCN_ERR_ARG, "null argument");
  *seg_out = nullptr; *n_out = 0; if (k_thresh) *k_thresh = 0.f; if (seg_min_verts) *seg_min_verts = 0; if (scene_id && scene_id_cap) scene_id[0] = 0;
  FILE* f = fopen(path, "rb");
  if (!f) return scn::fail(SCN_ERR_IO, "failed to open file %s", path);
  std::string buf; fseek(f, 0, SEEK_END); const long sz = ftell(f); fseek(f, 0, SEEK_SET);
  buf.resize(sz > 0 ? (size_t)sz : 0);
  const bool rd = buf.empty() || fread(&buf[0], 1, buf.size(), f) == buf.size(); fclose(f);
  if (!rd) return scn::fail(SCN_ERR_IO, "short read on %s", path);
  JsonCur c{buf.data(), buf.data() + buf.size(), {}};
  if (!c.eat('{')) return scn::fail(SCN_ERR_FORMAT, "Parse error reading %s at offset 0", path);
  std::vector<uint32_t> ids; bool have_ids = false;
  if (!c.eat('}')) for (;;) {
    std::string key;
    if (!c.str(key) || !c.eat(':')) return scn::fail(SCN_ERR_FORMAT, "Parse error reading %s at offset %zu", path, (size_t)(c.p - buf.data()));
    bool ok = true;
    if (key == "segIndices") {
      ok = c.eat('['); have_ids = ok;
      if (ok && !c.eat(']')) for (;;) {
        double v; c.ws();
        const bool is_null = c.e - c.p >= 4 && !strncmp(c.p, "null", 4);
        if (!c.num(v)) { ok = false; break; }
        ids.push_back(is_null ? 0xFFFFFFFFu : (v < 0 ? (uint32_t)(int32_t)v : (uint32_t)v));      // getUINT: (unsigned)GetInt() for negatives
        if (c.eat(',')) continue;
        ok = c.eat(']'); break;
      }
    } else if (key == "params") {
      ok = c.eat('{');
      if (ok && !c.eat('}')) for (;;) {
        std::string pk; double v;
        if (!c.str(pk) || !c.eat(':')) { ok = false; break; }
        if (pk == "kThresh") { ok = c.num(v); if (ok && k_thresh) *k_thresh = (float)v; }
        else if (pk == "segMinVerts") { ok = c.num(v); if (ok && seg_min_verts) *seg_min_verts = (uint32_t)v; }
        else ok = c.skip();
        if (!ok) break;
        if (c.eat(',')) continue;
        ok = c.eat('}'); break;
      }
    } else if (key == "sceneId") {
      std::string v; ok = c.str(v);
      if (ok && scene_id && scene_id_cap) { strncpy(scene_id, v.c_str(), scene_id_cap - 1); scene_id[scene_id_cap - 1] = 0; }
    } else ok = c.skip();
    if (!ok) return scn::fail(SCN_ERR_FORMAT, "Parse error reading %s at offset %zu", path, (size_t)(c.p - buf.data()));
    if (c.eat(',')) continue;
    if (!c.eat('}')) return scn::fail(SCN_ERR_FORMAT, "Parse error reading %s at offset %zu", path, (size_t)(c.p - buf.data()));
    break;
  }
  if (!have_ids) return scn::fail(SCN_ERR_FORMAT, "%s has no segIndices member", path);
  uint32_t* out = (uint32_t*)malloc(std::max<size_t>(ids.size(), 1) * 4);
  if (!out) return scn::fail(SCN_ERR_ARG, "out of memory");
  if (!ids.empty()) memcpy(out, ids.data(), ids.size() * 4);
  *seg_out = out; *n_out = ids.size();
  return SCN_OK;
}

// one mesh: segmentator.cpp:268-288 (same stdout lines, file naming); the caller has started the CUDA context warm-up
static int segment_one_file(const std::string& plyFile, float kthr, int segMinVerts, std::thread* warm) {
  printf("Segmenting %s with kThresh=%f, segMinVerts=%d ...\n", plyFile.c_str(), kthr, segMinVerts);
  const bool timing = getenv("SCN_TIMING") != nullptr;
  auto now = []() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
  const double t_start = now();
  float* xyz = nullptr; uint32_t* tri = nullptr; uint64_t nV = 0, nF = 0;
  const int load_rc = scn_mesh_load(plyFile.c_str(), &xyz, &nV, &tri, &nF);
  if (warm && warm->joinable()) warm->join();
  if (load_rc) { std::cerr << scn_last_error() << std::endl; return 1; }
  printf("Read mesh with vertexCount %lu %lu, faceCount %lu %lu\n", (unsigned long)nV, (unsigned long)(nV * 3), (unsigned long)nF, (unsigned long)(nF * 3));
  const double t_loaded = now();
  std::vector<int32_t> comps(nV);
  if (scn_segment_mesh(xyz, nV, tri, nF, kthr, segMinVerts, comps.data(), 0)) { std::cerr << scn_last_error() << std::endl; scn_free(xyz); scn_free(tri); return 1; }
  scn_free(xyz); scn_free(tri);
  const double t_segmented = now();
  // number of distinct ids (the reference fills an unordered_set, segmentator.cpp:279-282); ids are vertex indices < nV
  std::vector<uint8_t> seen(nV ? nV : 1, 0); size_t n_ids = 0;
  for (int32_t c : comps) if (!seen[(size_t)c]) { seen[(size_t)c] = 1; ++n_ids; }
  const std::string baseName = plyFile.substr(0, plyFile.find_last_of("."));
  const int lastslash = (int)plyFile.find_last_of("/");
  const std::string scanId = lastslash > 0 ? baseName.substr(lastslash) : baseName;
  const std::string segFile = baseName + "." + std::to_string(kthr) + ".segs.json";
  if (scn_write_segs_json(segFile.c_str(), scanId.c_str(), kthr, segMinVerts, comps.data(), comps.size())) { std::cerr << scn_last_error() << std::endl; return 1; }
  if (timing) {
    float ms[8]; scn_segment_last_timings(ms);
    fprintf(stderr, "[timing] load %.3f s, segment %.3f s (h2d %.1f normals %.1f weights %.1f sort %.1f kruskal %.1f small %.1f prune+d2h+labels %.1f ms), json+count %.3f s\n",
            t_loaded - t_start, t_segmented - t_loaded, ms[0], ms[1], ms[2], ms[3], ms[4], ms[5], ms[6], now() - t_segmented);
  }
  printf("Segmentation written to %s with %lu segments\n", segFile.c_str(), (unsigned long)n_ids);
  return 0;
}

// `segmentator input.ply [kThresh] [segMinVerts]` as the reference; plus `segmentator --batch list.txt [kThresh] [segMinVerts]`:
// every mesh named in list.txt (one path per line) in ONE process, so that the ~0.3 s of CUDA context creation - several
// times the reference's whole run on a 50 k-vertex mesh - is paid once per batch instead of once per mesh
// (Server/scan_processor.py:156 calls the tool once per scan; a batch is what a re-processing job wants).
int scn_segmentator_main(int argc, const char** argv) {
  if (argc < 2) {
    printf("Usage: ./segmentator input.ply [kThresh] [segMinVerts] (defaults: kThresh=0.01 segMinVerts=20)\n");
    return 255;                                                          // exit(-1)
  }
  std::thread warm([]() { scn_cuda_warmup(); });          // context creation overlaps the file read
  if (!strcmp(argv[1], "--batch")) {
    if (argc < 3) { warm.join(); printf("Usage: ./segmentator --batch list.txt [kThresh] [segMinVerts]\n"); return 255; }
    const float kthr = argc > 3 ? (float)atof(argv[3]) : 0.01f;
    const int segMinVerts = argc > 4 ? atoi(argv[4]) : 20;
    std::ifstream lf(argv[2]);
    if (!lf) { warm.join(); std::cerr << "cannot open " << argv[2] << std::endl; return 1; }
    std::string line; int rc = 0;
    while (std::getline(lf, line)) {
      while (!line.empty() && (line.back() == '\r' || line.back() == ' ')) line.pop_back();
      if (line.empty()) continue;
      rc |= segment_one_file(line, kthr, segMinVerts, &warm);
    }
    if (warm.joinable()) warm.join();
    return rc;
  }
  const std::string plyFile = argv[1];
  const float kthr = argc > 2 ? (float)atof(argv[2]) : 0.01f;
  const int segMinVerts = argc > 3 ? atoi(argv[3]) : 20;
  const int rc = segment_one_file(plyFile, kthr, segMinVerts, &warm);
  if (warm.joinable()) warm.join();
  return rc;
}

int scn_mesh_save_ply(const char* path, const float* xyz, const uint8_t* rgb, uint64_t n_verts, const uint32_t* tri, uint64_t n_faces) {
  if (!path || (!xyz && n_verts) || (!tri && n_faces)) return scn::fail(SCN_ERR_ARG, "null argument");
  char head[512];
  const int hl = snprintf(head, sizeof(head),
             "ply\nformat binary_little_endian 1.0\ncomment VCGLIB generated\nelement vertex %llu\nproperty float x\nproperty float y\nproperty float z\n"
             "property uchar red\nproperty uchar green\nproperty uchar blue\nproperty uchar alpha\nelement face %llu\nproperty list uchar int vertex_indices\nend_header\n",
          (unsigned long long)n_verts, (unsigned long long)n_faces);
  const size_t vbytes = (size_t)n_verts * 16, fbytes = (size_t)n_faces * 13, total = (size_t)hl + vbytes + fbytes;
  // records are written by a few threads straight into the mapped output file (a 5.7 M-vertex mesh is 240 MB: building it in a
  // buffer and fwrite-ing it was one thread at 1.3 GB/s); a plain buffered write is the fallback where the file cannot be mapped
  auto fill = [&](uint8_t* base, size_t lo, size_t hi) {            // bytes [lo, hi) of the body, on record boundaries
    for (size_t i = lo / 16; i < std::min<size_t>(n_verts, (hi + 15) / 16) && lo < vbytes; ++i) {
      uint8_t* r = base + i * 16;
      memcpy(r, xyz + 3 * i, 12);
      if (rgb) { r[12] = rgb[3 * i]; r[13] = rgb[3 * i + 1]; r[14] = rgb[3 * i + 2]; } else r[12] = r[13] = r[14] = 255;
      r[15] = 255;
    }
    (void)hi;
  };
  const int fd = ::open(path, O_RDWR | O_CREAT | O_TRUNC, 0644);
  if (fd < 0) return scn::fail(SCN_ERR_IO, "cannot write %s", path);
  bool ok = false;
  if (total > (size_t)(1 << 20) && ftruncate(fd, (off_t)total) == 0) {
    void* m = mmap(nullptr, total, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
    if (m != MAP_FAILED) {
      uint8_t* base = (uint8_t*)m;
      memcpy(base, head, (size_t)hl);
      uint8_t* vb = base + hl; uint8_t* fb = vb + vbytes;
      const unsigned nt = std::max(1u, std::min(16u, std::thread::hardware_concurrency()));
      auto work = [&](unsigned t) {
        const size_t v0 = (size_t)n_verts * t / nt, v1 = (size_t)n_verts * (t + 1) / nt;
        fill(vb, v0 * 16, v1 * 16);
        const size_t f0 = (size_t)n_faces * t / nt, f1 = (size_t)n_faces * (t + 1) / nt;
        for (size_t i = f0; i < f1; ++i) { fb[i * 13] = 3; memcpy(fb + i * 13 + 1, tri + 3 * i, 12); }
      };
      std::vector<std::thread> th;
      for (unsigned t = 1; t < nt; ++t) th.emplace_back(work, t);
      work(0);
      for (auto& x : th) x.join();
      ok = munmap(m, total) == 0;
      ::close(fd);
      return ok ? SCN_OK : scn::fail(SCN_ERR_IO, "short write on %s", path);
    }
    if (ftruncate(fd, 0) != 0) { ::close(fd); return scn::fail(SCN_ERR_IO, "cannot write %s", path); }
  }
  FILE* f = fdopen(fd, "wb");
  if (!f) { ::close(fd); return scn::fail(SCN_ERR_IO, "cannot write %s", path); }
  ok = fwrite(head, 1, (size_t)hl, f) == (size_t)hl;
  std::vector<uint8_t> buf(vbytes);
  fill(buf.data(), 0, vbytes);
  ok = ok && fwrite(buf.data(), 1, buf.size(), f) == buf.size();
  buf.resize(fbytes);
  for (uint64_t i = 0; i < n_faces; ++i) { buf[i * 13] = 3; memcpy(&buf[i * 13 + 1], tri + 3 * i, 12); }
  ok = ok && fwrite(buf.data(), 1, buf.size(), f) == buf.size();
  ok = (fclose(f) == 0) && ok;
  return ok ? SCN_OK : scn::fail(SCN_ERR_IO, "short write on %s", path);
}

}  // extern "C"
