// Mesh cleaning, host side: the MeshLab FilterScript reader and the `meshclean` command line (the kernels are in meshclean.cu).
//
//   scn_mesh_clean_params_from_mlx   reads the filters of Server/tools/meshclean/clean.mlx and cleanLoRes.mlx
//   scn_meshclean_main               `meshclean -i in.ply -o out.ply [-m vc] [-s script.mlx]`, the meshlabserver arguments of
//                                    Server/scan_processor.py:134,143
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

}  // namespace

extern "C" {

int scn_mesh_clean_params_from_mlx(const char* path, scn_mesh_clean_params* p) {
  if (!path || !p) return scn::fail(SCN_ERR_ARG, "null argument");
  std::ifstream in(path, std::ios::binary);
  if (!in) return scn::fail(SCN_ERR_IO, "cannot open %s", path);
  std::stringstream ss; ss << in.rdbuf();
  const std::string xml = ss.str();
  if (xml.find("<FilterScript") == std::string::npos) return scn::fail(SCN_ERR_FORMAT, "%s is not a MeshLab FilterScript", path);
  scn_mesh_clean_params q = *p;
  bool seen[4] = {false, false, false, false};
  int last = -1;
  std::string cur;                                   // the filter whose <Param> tags follow
  size_t pos = 0;
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
  float* xyz = nullptr; uint8_t* rgb = nullptr; uint32_t* tri = nullptr; uint64_t nV = 0, nF = 0;
  const int lrc = scn_mesh_load_rgb(in, &xyz, &rgb, &nV, &tri, &nF);
  warm.join();
  if (lrc) { fprintf(stderr, "%s\n", scn_last_error()); return 1; }
  printf("Loaded %s: %llu vertices, %llu faces%s\n", in, (unsigned long long)nV, (unsigned long long)nF, rgb ? ", vertex colour" : "");
  float* oxyz = nullptr; uint8_t* orgb = nullptr; uint32_t* otri = nullptr; uint64_t oV = 0, oF = 0;
  scn_mesh_clean_report_t r;
  const int crc = scn_mesh_clean(xyz, vc ? rgb : nullptr, nV, tri, nF, &p, &oxyz, &orgb, &otri, &oV, &oF, &r);
  scn_free(xyz); scn_free(rgb); scn_free(tri);
  if (crc) { fprintf(stderr, "%s\n", scn_last_error()); return 1; }
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
  const int src = scn_mesh_save_ply(out, oxyz, orgb, oV, otri, oF);
  scn_free(oxyz); scn_free(orgb); scn_free(otri);
  if (src) { fprintf(stderr, "%s\n", scn_last_error()); return 1; }
  printf("Saved %s: %llu vertices, %llu faces\n", out, (unsigned long long)oV, (unsigned long long)oF);
  return 0;
}

}  // extern "C"
