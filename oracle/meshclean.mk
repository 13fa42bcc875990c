# TEST INFRASTRUCTURE.  The mesh-cleaning oracles (DESIGN.md §6f), beside oracle/Makefile and in its style:
#   (1) this repo's sequential restatement, oracle/meshclean_oracle.c -> _build/liboracle_meshclean.so, and
#   (2) the UNMODIFIED mLib MeshData (mergeCloseVertices, removeDuplicateFaces), meshData.h + meshData.cpp compiled where they
#       lie behind ref_shim_meshdata.cpp -> _ref/libref_meshdata.so (only where the reference tree exists).
# Run from oracle/:  make -f meshclean.mk all   (the top-level Makefile's `oracle` target and __graft_entry__.build() do).
REF      ?= /root/reference
CXX      := $(if $(wildcard /usr/bin/g++),/usr/bin/g++,g++)
CC       := $(if $(wildcard /usr/bin/gcc),/usr/bin/gcc,gcc)
REFOUT   := _ref
OUT      := _build

all: oracle ref
oracle: $(OUT)/liboracle_meshclean.so

$(OUT)/liboracle_meshclean.so: meshclean_oracle.c | $(OUT)
	$(CC) -std=c11 -O2 -ffp-contract=off -fPIC -shared -o $@ $< -lm

$(OUT) $(REFOUT):
	mkdir -p $@

ifneq ($(wildcard $(REF)/external/mLib/include/core-mesh/meshData.cpp),)
ref: $(REFOUT)/libref_meshdata.so
$(REFOUT)/libref_meshdata.so: ref_shim_meshdata.cpp | $(REFOUT)
	$(CXX) -std=c++17 -O2 -ffp-contract=off -w -fPIC -shared -I$(REF)/external/mLib/include -o $@ ref_shim_meshdata.cpp
else
ref:
	@echo "reference tree not present; using prebuilt $(REFOUT)/libref_meshdata.so if any"
endif

.PHONY: all oracle ref
