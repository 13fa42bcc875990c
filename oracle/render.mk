# TEST INFRASTRUCTURE.  The render oracle (DESIGN.md §6i), beside freespace.mk and in its style:
#   oracle/render_oracle.c -> _build/liboracle_render.so, this repo's scalar statement of its own spec (Mitsuba, which the
#   reference pipeline's `render` stage drives through Server/mts_render.py, is not in the reference tree).
# Run from oracle/:  make -f render.mk all   (the top-level Makefile's `oracle` target and __graft_entry__.build() do).
CC       := $(if $(wildcard /usr/bin/gcc),/usr/bin/gcc,gcc)
OUT      := _build

all: $(OUT)/liboracle_render.so

$(OUT)/liboracle_render.so: render_oracle.c | $(OUT)
	$(CC) -std=c11 -O2 -Wall -ffp-contract=off -fopenmp -fPIC -shared -o $@ $< -lm

$(OUT):
	mkdir -p $@

.PHONY: all
