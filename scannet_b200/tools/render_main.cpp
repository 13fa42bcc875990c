// `render [options] mesh.ply` — drop-in for `python mts_render.py <id>_vh_clean_2.ply` of
// /root/reference/Server/scan_processor.py:158-160 (the `render` stage): writes <id>_vh_clean_2.png beside the input.
#include "scannet_b200.h"
int main(int argc, const char** argv) { return scn_render_main(argc, argv); }
