# TEST INFRASTRUCTURE.  The free-space oracle (DESIGN.md §6h), beside meshclean.mk and meshsimplify.mk and in their style:
#   oracle/freespace_oracle.c -> _build/liboracle_freespace.so, this repo's scalar statement of its own spec (FreeSpace.exe,
#   the reference pipeline's `freespace` binary, is not in the reference tree).  -mfma: fmaf must be one fused operation.
# Run from oracle/:  make -f freespace.mk all   (the top-level Makefile's `oracle` target and __graft_entry__.build() do).
CC       := $(if $(wildcard /usr/bin/gcc),/usr/bin/gcc,gcc)
OUT      := _build

all: $(OUT)/liboracle_freespace.so

$(OUT)/liboracle_freespace.so: freespace_oracle.c | $(OUT)
	$(CC) -std=c11 -O2 -Wall -ffp-contract=off -mfma -fopenmp -fPIC -shared -o $@ $< -lm

$(OUT):
	mkdir -p $@

.PHONY: all
