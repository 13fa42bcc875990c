# TEST INFRASTRUCTURE.  The decimation oracle (DESIGN.md §6g), beside meshclean.mk and in its style:
#   oracle/meshsimplify_oracle.c -> _build/liboracle_meshsimplify.so, this repo's sequential statement of its own spec (no
#   reference code exists for quadric edge collapse: MeshLab/VCG is not in the reference tree).
# Run from oracle/:  make -f meshsimplify.mk all   (the top-level Makefile's `oracle` target and __graft_entry__.build() do).
CC       := $(if $(wildcard /usr/bin/gcc),/usr/bin/gcc,gcc)
OUT      := _build

all: $(OUT)/liboracle_meshsimplify.so

$(OUT)/liboracle_meshsimplify.so: meshsimplify_oracle.c | $(OUT)
	$(CC) -std=c11 -O2 -Wall -ffp-contract=off -fPIC -shared -o $@ $< -lm

$(OUT):
	mkdir -p $@

.PHONY: all
