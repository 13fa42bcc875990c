// TEST INFRASTRUCTURE — not product code.
//
// C-callable shim around the UNMODIFIED mLib MeshData of the reference tree
// (/root/reference/external/mLib/include/core-mesh/meshData.h + meshData.cpp), compiled where it lies by oracle/meshclean.mk into
// oracle/_ref/libref_meshdata.so.  MeshData normally comes in through mLibCore.h, which needs the whole (Windows-oriented)
// library; the names its declarations mention but the two operators under test never use are declared empty below.
//
//   ref_mesh_clean   MeshData<float>::mergeCloseVertices(t, false)   meshData.cpp:217-289 (incl. removeDegeneratedFaces :293-318)
//                    MeshData<float>::removeDuplicateFaces()          meshData.cpp:40-104
// removeIsolatedPieces / removeIsolatedVertices are not here: meshData.cpp:335 binds a non-const reference to the Face
// temporary that Indices' iterator returns, which g++ rejects.
#include <algorithm>
#include <cassert>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <iostream>
#include <list>
#include <map>
#include <set>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <vector>
#define LINUX
#include "core-base/common.h"
namespace ml {
template <class T> class BinaryDataSerialize {};
template <class A, class B> class BinaryDataStream {};
template <class T> class Matrix4x4 {};
template <class T> class Matrix3x3 {};
template <class T> class BoundingBox3 {};
template <class T> class Plane {};
template <class T> class Material { public: std::string m_name; };
}  // namespace ml
#include "core-util/utility.h"
#include "core-util/stringUtil.h"
#include "core-math/vec1.h"
#include "core-math/vec2.h"
#include "core-math/vec3.h"
#include "core-math/vec4.h"
#include "core-util/sparseGrid3.h"
#include "core-mesh/meshData.h"

extern "C" {

// steps: bit0 = mergeCloseVertices(t, false), bit1 = removeDuplicateFaces, in that order.  Colours travel as vec4<float>
// holding the byte values (u8 -> float -> u8 is exact).  Outputs are caller-owned with room for nV / nF.
// Returns 0, or -1 when mLib throws.
int ref_mesh_clean(const float* xyz, const uint8_t* rgb, int64_t nV, const uint32_t* tri, int64_t nF, float t, int steps,
                   float* xyz_out, uint8_t* rgb_out, uint32_t* tri_out, int64_t* nV_out, int64_t* nF_out) {
  ml::MeshDataf m;
  for (int64_t i = 0; i < nV; ++i) m.m_Vertices.push_back(ml::vec3f(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]));
  if (rgb) for (int64_t i = 0; i < nV; ++i) m.m_Colors.push_back(ml::vec4f((float)rgb[3 * i], (float)rgb[3 * i + 1], (float)rgb[3 * i + 2], 255.f));
  for (int64_t f = 0; f < nF; ++f) m.m_FaceIndicesVertices.addFace(tri + 3 * f, 3);
  try {
    if (steps & 1) m.mergeCloseVertices(t, false);
    if (steps & 2) m.removeDuplicateFaces();
  } catch (...) {
    return -1;
  }
  *nV_out = (int64_t)m.m_Vertices.size();
  for (size_t i = 0; i < m.m_Vertices.size(); ++i) {
    xyz_out[3 * i] = m.m_Vertices[i].x; xyz_out[3 * i + 1] = m.m_Vertices[i].y; xyz_out[3 * i + 2] = m.m_Vertices[i].z;
    if (rgb) for (int k = 0; k < 3; ++k) rgb_out[3 * i + k] = (uint8_t)m.m_Colors[i][k];
  }
  *nF_out = (int64_t)m.m_FaceIndicesVertices.size();
  for (size_t f = 0; f < m.m_FaceIndicesVertices.size(); ++f) {
    const auto& face = m.m_FaceIndicesVertices[f];
    for (int k = 0; k < 3; ++k) tri_out[3 * f + k] = face[k];
  }
  return 0;
}

}  // extern "C"
