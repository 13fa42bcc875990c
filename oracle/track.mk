# TEST INFRASTRUCTURE.  The tracker oracle (DESIGN.md §6j), beside render.mk and in its style:
#   oracle/track_oracle.c -> _build/liboracle_track.so, this repo's scalar statement of its own tracking spec (BundleFusion, which the
#   reference pipeline's `recons` stage runs through Server/scan_processor.py, is not in the reference tree).  It includes
#   tsdf_oracle.c, so the whole loop (track -> integrate -> raycast) runs on the CPU; -mfma as for liboracle_tsdf.so (fmaf fused).
# Run from oracle/:  make -f track.mk all   (the top-level Makefile's `oracle` target and __graft_entry__.build() do).
CC       := $(if $(wildcard /usr/bin/gcc),/usr/bin/gcc,gcc)
OUT      := _build

all: $(OUT)/liboracle_track.so

$(OUT)/liboracle_track.so: track_oracle.c tsdf_oracle.c | $(OUT)
	$(CC) -std=c11 -O2 -Wall -Wno-unused-function -ffp-contract=off -mfma -fopenmp -fPIC -shared -o $@ $< -lm

$(OUT):
	mkdir -p $@

.PHONY: all
