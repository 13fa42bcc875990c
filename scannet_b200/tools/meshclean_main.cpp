// `meshclean -i in.ply -o out.ply [-m vc] [-s clean.mlx]` — drop-in for the `meshlabserver ... -s clean.mlx` call of
// /root/reference/Server/scan_processor.py:143 (decimate1).
#include "scannet_b200.h"
int main(int argc, const char** argv) { return scn_meshclean_main(argc, argv); }
