// `recons <params.txt> <params2.txt> <file.sens> [out.ply]` — drop-in for the `FriedLiver.exe` call of
// /root/reference/Server/scan_processor.py:27-29,123-126 (the `recons` stage): tracks the stream, writes <base>.ply beside the input
// and the trajectory back into the .sens.  A frame-to-model tracker, not BundleFusion (DESIGN.md §6j).
#include "scannet_b200.h"
int main(int argc, const char** argv) { return scn_recons_main(argc, argv); }
