// Mesh cleaning and decimation, host side: the MeshLab FilterScript readers and the `meshclean` / `meshsimplify` command lines
// (the kernels are in meshclean.cu and meshsimplify.cu).
//
//   scn_mesh_clean_params_from_mlx      reads the filters of Server/tools/meshclean/clean.mlx and cleanLoRes.mlx
//   scn_mesh_simplify_params_from_mlx   reads simplify.mlx: Quadric Edge Collapse Decimation, then clean.mlx's filters
//   scn_meshclean_main                  `meshclean -i in.ply -o out.ply [-m vc] [-s script.mlx]`, the meshlabserver arguments of
//                                       Server/scan_processor.py:134,143
//   scn_meshsimplify_main               `meshsimplify -i in.ply -o out.ply [-m vc] [-s simplify.mlx]`, scan_processor.py:144-145
#include <chrono>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <sstream>
#include <string>
#include <thread>
#include <vector>

#include "scn_common.h"

namespace {

// value of attribute `name` inside one XML start tag (quotes ' or "); false when absent
bool xml_attr(const std::string& tag, const char* name, std::string& out) {
  const std::string key = std::string(name) + "=";
  size_t p = 0;
  while ((p = tag.find(key, p)) != std::string::npos) {
    if (p > 0 && !isspace((unsigned char)tag[p - 1])) { p += key.size(); continue; }
    const size_t q = p + key.size();
    if (q >= tag.size() || (tag[q] != '"' && tag[q] != '\'')) return false;
    const size_t e = tag.find(tag[q], q + 1);
    if (e == std::string::npos) return false;
    out = tag.substr(q + 1, e - q - 1);
    return true;
  }
  return false;
}

// the clean.mlx filters, in the order the stage runs them
const char* const kFilters[] = {"Merge Close Vertices", "Remove Duplicate Faces", "Remove Isolated pieces (wrt Face Num.)",
                                "Remove Unreferenced Vertex"};

// reads clean.mlx's filters from the tag at `pos` on into *p (unchanged on error)
int parse_clean(const std::string& xml, size_t pos, const char* path, scn_mesh_clean_params* p) {
  scn_mesh_clean_params q = *p;
  bool seen[4] = {false, false, false, false};
  int last = -1;
  std::string cur;                                   // the filter whose <Param> tags follow
  while ((pos = xml.find('<', pos)) != std::string::npos) {
    const size_t end = xml.find('>', pos);
    if (end == std::string::npos) return scn::fail(SCN_ERR_FORMAT, "%s: unterminated tag", path);
    const std::string tag = xml.substr(pos + 1, end - pos - 1);
    pos = end + 1;
    if (tag.compare(0, 7, "filter ") == 0 || tag.compare(0, 7, "filter\t") == 0) {
      std::string name;
      if (!xml_attr(tag, "name", name)) return scn::fail(SCN_ERR_FORMAT, "%s: a filter without a name", path);
      int k = -1;
      for (int i = 0; i < 4; ++i) if (name == kFilters[i]) k = i;
      if (k < 0) return scn::fail(SCN_ERR_UNSUPPORTED, "%s: filter \"%s\" is not supported (only the filters of clean.mlx: Merge Close Vertices, "
                                  "Remove Duplicate Faces, Remove Isolated pieces (wrt Face Num.), Remove Unreferenced Vertex)", path, name.c_str());
      if (seen[k] || k < last)
        return scn::fail(SCN_ERR_UNSUPPORTED, "%s: filter \"%s\" repeated or out of clean.mlx's order", path, name.c_str());
      seen[k] = true; last = k; cur = name;
    } else if (tag.compare(0, 6, "Param ") == 0 || tag.compare(0, 6, "Param\t") == 0) {
      std::string name, value;
      if (!xml_attr(tag, "name", name) || !xml_attr(tag, "value", value)) return scn::fail(SCN_ERR_FORMAT, "%s: a Param without name or value", path);
      char* e = nullptr;
      if (cur == kFilters[0] && name == "Threshold") {
        const double t = strtod(value.c_str(), &e);
        if (e == value.c_str() || *e) return scn::fail(SCN_ERR_FORMAT, "%s: Threshold \"%s\" is not a number", path, value.c_str());
        q.merge_threshold = (float)t;
      } else if (cur == kFilters[2] && name == "MinComponentSize") {
        const long long n = strtoll(value.c_str(), &e, 10);
        if (e == value.c_str() || *e || n < 0 || n > 0xFFFFFFFFll) return scn::fail(SCN_ERR_FORMAT, "%s: MinComponentSize \"%s\" is not a count", path, value.c_str());
        q.min_piece_faces = (uint32_t)n;
      }
    }
  }
  q.flags &= ~(SCN_CLEAN_SKIP_MERGE | SCN_CLEAN_SKIP_DEDUP | SCN_CLEAN_SKIP_PIECES);
  if (!seen[0]) q.flags |= SCN_CLEAN_SKIP_MERGE;
  if (!seen[1]) q.flags |= SCN_CLEAN_SKIP_DEDUP;
  if (!seen[2] && !seen[3]) q.flags |= SCN_CLEAN_SKIP_PIECES;
  if (!seen[2]) { q.min_piece_faces = 0; q.min_piece_vertices = 0; }   // Remove Unreferenced Vertex alone: compaction only
  *p = q;
  return SCN_OK;
}

// the '>' that closes the tag opened at `pos`, skipping quoted attribute values (simplify.mlx's tooltips hold "&lt;br>")
size_t tag_end(const std::string& xml, size_t pos) {
  char quote = 0;
  for (size_t i = pos + 1; i < xml.size(); ++i) {
    const char c = xml[i];
    if (quote) { if (c == quote) quote = 0; }
    else if (c == '"' || c == '\'') quote = c;
    else if (c == '>') return i;
  }
  return std::string::npos;
}

// the lines of the clean filters that ran: their counters, and the size of the mesh they left
void print_clean(const scn_mesh_clean_params& p, const scn_mesh_clean_report_t& r, uint64_t oV, uint64_t oF) {
  if (!(p.flags & SCN_CLEAN_SKIP_MERGE))
    printf("Merge Close Vertices (%g): %llu vertices merged, %llu degenerate faces removed (%.2f ms)\n", (double)p.merge_threshold,
           (unsigned long long)r.vertices_merged, (unsigned long long)r.degenerate_faces, r.merge_ms);
  if (!(p.flags & SCN_CLEAN_SKIP_DEDUP))
    printf("Remove Duplicate Faces: %llu faces removed (%.2f ms)\n", (unsigned long long)r.duplicate_faces, r.dedup_ms);
  if (!(p.flags & SCN_CLEAN_SKIP_PIECES)) {
    printf("Remove Isolated pieces (min %u faces, %u vertices): %llu of %llu pieces removed, %llu faces (%.2f ms)\n", p.min_piece_faces,
           p.min_piece_vertices, (unsigned long long)r.pieces_removed, (unsigned long long)r.pieces_total,
           (unsigned long long)r.faces_in_removed_pieces, r.pieces_ms);
    printf("Remove Unreferenced Vertex: %llu vertices, %llu faces remain\n", (unsigned long long)oV, (unsigned long long)oF);
  }
}

bool read_file(const char* path, std::string& xml) {
  std::ifstream in(path, std::ios::binary);
  if (!in) return false;
  std::stringstream ss; ss << in.rdbuf();
  xml = ss.str();
  return true;
}

}  // namespace

extern "C" {

int scn_mesh_clean_params_from_mlx(const char* path, scn_mesh_clean_params* p) {
  if (!path || !p) return scn::fail(SCN_ERR_ARG, "null argument");
  std::string xml;
  if (!read_file(path, xml)) return scn::fail(SCN_ERR_IO, "cannot open %s", path);
  if (xml.find("<FilterScript") == std::string::npos) return scn::fail(SCN_ERR_FORMAT, "%s is not a MeshLab FilterScript", path);
  return parse_clean(xml, 0, path, p);
}

int scn_meshclean_main(int argc, const char** argv) {
  const char* in = nullptr; const char* out = nullptr; const char* script = nullptr;
  bool vc = false;
  for (int i = 1; i < argc; ++i) {
    const std::string a = argv[i];
    if ((a == "-i" || a == "-o" || a == "-s" || a == "-m") && i + 1 < argc) {
      const char* v = argv[++i];
      if (a == "-i") in = v; else if (a == "-o") out = v; else if (a == "-s") script = v;
      else vc = vc || std::strstr(v, "vc") != nullptr;             // -m vc: keep vertex colour
    } else {
      fprintf(stderr, "meshclean: unexpected argument %s\n", argv[i]);
      in = nullptr; break;
    }
  }
  if (!in || !out) {
    printf("Usage: meshclean -i in.ply -o out.ply [-m vc] [-s script.mlx]   (without -s: the clean.mlx defaults)\n");
    return 255;
  }
  std::thread warm([]() { scn_cuda_warmup(); });
  scn_mesh_clean_params p;
  scn_mesh_clean_default_params(&p);
  if (script && scn_mesh_clean_params_from_mlx(script, &p)) { warm.join(); fprintf(stderr, "%s\n", scn_last_error()); return 1; }
  float* x = nullptr; uint8_t* c = nullptr; uint32_t* t = nullptr; uint64_t nV = 0, nF = 0;
  const int lrc = scn_mesh_load_rgb(in, &x, &c, &nV, &t, &nF);
  const scn::MallocPtr<float> xyz(x); const scn::MallocPtr<uint8_t> rgb(c); const scn::MallocPtr<uint32_t> tri(t);
  warm.join();
  if (lrc) { fprintf(stderr, "%s\n", scn_last_error()); return 1; }
  printf("Loaded %s: %llu vertices, %llu faces%s\n", in, (unsigned long long)nV, (unsigned long long)nF, rgb ? ", vertex colour" : "");
  float* ox = nullptr; uint8_t* oc = nullptr; uint32_t* ot = nullptr; uint64_t oV = 0, oF = 0;
  scn_mesh_clean_report_t r;
  const int crc = scn_mesh_clean(xyz.get(), vc ? rgb.get() : nullptr, nV, tri.get(), nF, &p, &ox, &oc, &ot, &oV, &oF, &r);
  const scn::MallocPtr<float> oxyz(ox); const scn::MallocPtr<uint8_t> orgb(oc); const scn::MallocPtr<uint32_t> otri(ot);
  if (crc) { fprintf(stderr, "%s\n", scn_last_error()); return 1; }
  print_clean(p, r, oV, oF);
  if (scn_mesh_save_ply(out, oxyz.get(), orgb.get(), oV, otri.get(), oF)) { fprintf(stderr, "%s\n", scn_last_error()); return 1; }
  printf("Saved %s: %llu vertices, %llu faces\n", out, (unsigned long long)oV, (unsigned long long)oF);
  return 0;
}

int scn_mesh_simplify_params_from_mlx(const char* path, scn_mesh_simplify_params* p, scn_mesh_clean_params* after) {
  if (!path || !p || !after) return scn::fail(SCN_ERR_ARG, "null argument");
  std::string xml;
  if (!read_file(path, xml)) return scn::fail(SCN_ERR_IO, "cannot open %s", path);
  if (xml.find("<FilterScript") == std::string::npos) return scn::fail(SCN_ERR_FORMAT, "%s is not a MeshLab FilterScript", path);
  static const char* const kQuadric = "Quadric Edge Collapse Decimation";
  // simplify.mlx's values of the options that are not implemented (1 = true, 0 = false; BoundaryWeight must be 1)
  static const struct { const char* name; int value; } kFixed[] = {
      {"PreserveBoundary", 0}, {"PreserveNormal", 0}, {"PreserveTopology", 0}, {"OptimalPlacement", 1},
      {"PlanarQuadric", 0},    {"QualityWeight", 0},  {"AutoClean", 1},        {"Selected", 0}};
  scn_mesh_simplify_params q = *p;
  bool in_quadric = false, seen = false;
  size_t pos = 0;
  while ((pos = xml.find('<', pos)) != std::string::npos) {
    const size_t end = tag_end(xml, pos);
    if (end == std::string::npos) return scn::fail(SCN_ERR_FORMAT, "%s: unterminated tag", path);
    const std::string tag = xml.substr(pos + 1, end - pos - 1);
    if (tag.compare(0, 7, "filter ") == 0 || tag.compare(0, 7, "filter\t") == 0) {
      std::string name;
      if (!xml_attr(tag, "name", name)) return scn::fail(SCN_ERR_FORMAT, "%s: a filter without a name", path);
      if (name != kQuadric || seen) {
        if (!seen) return scn::fail(SCN_ERR_UNSUPPORTED, "%s: the first filter must be \"%s\", not \"%s\"", path, kQuadric, name.c_str());
        break;                                     // the clean filters from here on (a second decimation is refused there)
      }
      seen = in_quadric = true;
    } else if (in_quadric && (tag.compare(0, 6, "Param ") == 0 || tag.compare(0, 6, "Param\t") == 0)) {
      std::string name, value;
      if (!xml_attr(tag, "name", name) || !xml_attr(tag, "value", value)) return scn::fail(SCN_ERR_FORMAT, "%s: a Param without name or value", path);
      char* e = nullptr;
      if (name == "TargetFaceNum") {
        const long long n = strtoll(value.c_str(), &e, 10);
        if (e == value.c_str() || *e || n < 0) return scn::fail(SCN_ERR_FORMAT, "%s: TargetFaceNum \"%s\" is not a count", path, value.c_str());
        q.target_faces = (uint64_t)n;
      } else if (name == "TargetPerc" || name == "QualityThr" || name == "BoundaryWeight") {
        const double v = strtod(value.c_str(), &e);
        if (e == value.c_str() || *e) return scn::fail(SCN_ERR_FORMAT, "%s: %s \"%s\" is not a number", path, name.c_str(), value.c_str());
        if (name == "TargetPerc") q.target_perc = v;
        else if (name == "QualityThr") q.quality_thr = v;
        else if (v != 1.0) return scn::fail(SCN_ERR_UNSUPPORTED, "%s: BoundaryWeight %s is not supported (only 1)", path, value.c_str());
      } else {
        int k = -1;
        for (int i = 0; i < (int)(sizeof(kFixed) / sizeof(kFixed[0])); ++i) if (name == kFixed[i].name) k = i;
        if (k < 0) return scn::fail(SCN_ERR_UNSUPPORTED, "%s: parameter %s of %s is not supported", path, name.c_str(), kQuadric);
        const int v = value == "true" ? 1 : value == "false" ? 0 : -1;
        if (v != kFixed[k].value)
          return scn::fail(SCN_ERR_UNSUPPORTED, "%s: %s=%s is not supported (only %s)", path, name.c_str(), value.c_str(), kFixed[k].value ? "true" : "false");
      }
    }
    pos = end + 1;
  }
  if (!seen) return scn::fail(SCN_ERR_UNSUPPORTED, "%s: no \"%s\" filter", path, kQuadric);
  scn_mesh_clean_params a = *after;
  if (pos == std::string::npos) pos = xml.size();
  if (int rc = parse_clean(xml, pos, path, &a)) return rc;
  *p = q; *after = a;
  return SCN_OK;
}

int scn_meshsimplify_main(int argc, const char** argv) {
  const char* in = nullptr; const char* out = nullptr; const char* script = nullptr;
  bool vc = false;
  for (int i = 1; i < argc; ++i) {
    const std::string a = argv[i];
    if ((a == "-i" || a == "-o" || a == "-s" || a == "-m") && i + 1 < argc) {
      const char* v = argv[++i];
      if (a == "-i") in = v; else if (a == "-o") out = v; else if (a == "-s") script = v;
      else vc = vc || std::strstr(v, "vc") != nullptr;             // -m vc: keep vertex colour
    } else {
      fprintf(stderr, "meshsimplify: unexpected argument %s\n", argv[i]);
      in = nullptr; break;
    }
  }
  if (!in || !out) {
    printf("Usage: meshsimplify -i in.ply -o out.ply [-m vc] [-s simplify.mlx]   (without -s: the simplify.mlx defaults)\n");
    return 255;
  }
  std::thread warm([]() { scn_cuda_warmup(); });
  scn_mesh_simplify_params p;
  scn_mesh_clean_params c;
  scn_mesh_simplify_default_params(&p, &c);
  if (script && scn_mesh_simplify_params_from_mlx(script, &p, &c)) { warm.join(); fprintf(stderr, "%s\n", scn_last_error()); return 1; }
  float* x = nullptr; uint8_t* cl = nullptr; uint32_t* t = nullptr; uint64_t nV = 0, nF = 0;
  const int lrc = scn_mesh_load_rgb(in, &x, &cl, &nV, &t, &nF);
  const scn::MallocPtr<float> xyz(x); const scn::MallocPtr<uint8_t> rgb(cl); const scn::MallocPtr<uint32_t> tri(t);
  warm.join();
  if (lrc) { fprintf(stderr, "%s\n", scn_last_error()); return 1; }
  printf("Loaded %s: %llu vertices, %llu faces%s\n", in, (unsigned long long)nV, (unsigned long long)nF, rgb ? ", vertex colour" : "");
  float* ox = nullptr; uint8_t* oc = nullptr; uint32_t* ot = nullptr; uint64_t oV = 0, oF = 0;
  scn_mesh_simplify_report_t r;
  const int crc = scn_mesh_simplify(xyz.get(), vc ? rgb.get() : nullptr, nV, tri.get(), nF, &p, &c, &ox, &oc, &ot, &oV, &oF, &r);
  const scn::MallocPtr<float> oxyz(ox); const scn::MallocPtr<uint8_t> orgb(oc); const scn::MallocPtr<uint32_t> otri(ot);
  if (crc) { fprintf(stderr, "%s\n", scn_last_error()); return 1; }
  printf("Quadric Edge Collapse Decimation (target %llu faces, quality threshold %g): %llu collapses in %llu rounds removed %llu faces; "
         "AutoClean removed %llu duplicate faces, %llu vertices, %llu faces remain (%.2f ms)\n", (unsigned long long)r.target_faces,
         p.quality_thr, (unsigned long long)r.collapses, (unsigned long long)r.rounds, (unsigned long long)r.faces_collapsed,
         (unsigned long long)r.autoclean_duplicate_faces, (unsigned long long)r.clean.vertices_in, (unsigned long long)r.clean.faces_in,
         r.quadrics_ms + r.rounds_ms + r.autoclean_ms);
  print_clean(c, r.clean, oV, oF);
  if (scn_mesh_save_ply(out, oxyz.get(), orgb.get(), oV, otri.get(), oF)) { fprintf(stderr, "%s\n", scn_last_error()); return 1; }
  printf("Saved %s: %llu vertices, %llu faces\n", out, (unsigned long long)oV, (unsigned long long)oF);
  return 0;
}

}  // extern "C"
