// `freespace <file.sens>` — drop-in for the `FreeSpace.exe <file.sens>` call of /root/reference/Server/scan_processor.py:150-152
// (the `freespace` stage, Server/config/scan_stages.json:43-47): writes <base>.grid beside the input.
#include "scannet_b200.h"
int main(int argc, const char** argv) { return scn_freespace_main(argc, argv); }
