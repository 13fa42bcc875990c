# TEST INFRASTRUCTURE.  The global optimisation oracle (DESIGN.md §6k), beside track.mk and in its style:
#   oracle/globalopt_oracle.c -> _build/liboracle_globalopt.so, this repo's scalar statement of its dense keyframe optimisation (the
#   global stage of BundleFusion, which the reference pipeline's `recons` stage runs, is not in the reference tree).  It includes
#   track_oracle.c for the frame pipeline, the Cholesky solve and the Cayley update.
# Run from oracle/:  make -f globalopt.mk all   (the top-level Makefile's `oracle` target and __graft_entry__.build() do).
CC       := $(if $(wildcard /usr/bin/gcc),/usr/bin/gcc,gcc)
OUT      := _build

all: $(OUT)/liboracle_globalopt.so

$(OUT)/liboracle_globalopt.so: globalopt_oracle.c track_oracle.c tsdf_oracle.c | $(OUT)
	$(CC) -std=c11 -O2 -Wall -Wno-unused-function -ffp-contract=off -mfma -fopenmp -fPIC -shared -o $@ $< -lm

$(OUT):
	mkdir -p $@

.PHONY: all
