// `meshsimplify -i in.ply -o out.ply [-m vc] [-s simplify.mlx]` — drop-in for the two `meshlabserver ... -s simplify.mlx` calls
// of /root/reference/Server/scan_processor.py:144-145 (decimate2, decimate3).
#include "scannet_b200.h"
int main(int argc, const char** argv) { return scn_meshsimplify_main(argc, argv); }
