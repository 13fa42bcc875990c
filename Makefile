# Builds libscannet_b200.so (hand-written sm_90a CUDA for H100 behind the C ABI in include/scannet_b200.h),
# the host CLIs, and the test oracles.  nvcc cross-compiles without a GPU.
NVCC     ?= nvcc
ARCH     := -gencode arch=compute_90a,code=sm_90a
NVFLAGS  := -O3 -std=c++17 $(ARCH) -lineinfo -fmad=false -Xcompiler -fPIC,-Wall,-Wno-unused-function,-ffp-contract=off \
            -Xptxas -v --expt-relaxed-constexpr -ccbin /usr/bin/g++
CSRC     := scannet_b200/csrc
LIBDIR   := scannet_b200/lib
BINDIR   := scannet_b200/bin
OBJDIR   := build/obj
SRCS     := $(wildcard $(CSRC)/*.cu)
CPPSRCS  := $(wildcard $(CSRC)/*.cpp)
OBJS     := $(patsubst $(CSRC)/%.cu,$(OBJDIR)/%.o,$(SRCS)) $(patsubst $(CSRC)/%.cpp,$(OBJDIR)/%.cpp.o,$(CPPSRCS))
LIB      := $(LIBDIR)/libscannet_b200.so
TOOLS    := $(patsubst scannet_b200/tools/%_main.cpp,$(BINDIR)/%,$(wildcard scannet_b200/tools/*_main.cpp))

all: lib tools oracle
lib: $(LIB)
tools: $(TOOLS)

$(OBJDIR)/%.o: $(CSRC)/%.cu $(wildcard $(CSRC)/*.h) $(wildcard $(CSRC)/*.cuh) include/scannet_b200.h | $(OBJDIR)
	$(NVCC) $(NVFLAGS) -c $< -o $@ 2> $(OBJDIR)/$*.ptxas.log || (cat $(OBJDIR)/$*.ptxas.log; exit 1)

$(OBJDIR)/%.cpp.o: $(CSRC)/%.cpp $(wildcard $(CSRC)/*.h) include/scannet_b200.h | $(OBJDIR)
	/usr/bin/g++ -O3 -std=c++17 -fPIC -Wall -Wno-unused-function -Wno-misleading-indentation -ffp-contract=off -c $< -o $@

$(LIB): $(OBJS) | $(LIBDIR)
	$(NVCC) $(ARCH) -shared -o $@ $(OBJS) -ccbin /usr/bin/g++ -cudart static -lpthread

$(BINDIR)/%: scannet_b200/tools/%_main.cpp $(LIB) | $(BINDIR)
	/usr/bin/g++ -O2 -std=c++17 -Iinclude -o $@ $< -L$(LIBDIR) -lscannet_b200 -Wl,-rpath,'$$ORIGIN/../lib'

oracle:
	$(MAKE) -C oracle all
	$(MAKE) -C oracle -f meshclean.mk all
	$(MAKE) -C oracle -f meshsimplify.mk all
	$(MAKE) -C oracle -f freespace.mk all
	$(MAKE) -C oracle -f render.mk all
	$(MAKE) -C oracle -f track.mk all
	$(MAKE) -C oracle -f globalopt.mk all

$(OBJDIR) $(LIBDIR) $(BINDIR):
	mkdir -p $@

clean:
	rm -rf build $(LIBDIR) $(BINDIR) oracle/_build
.PHONY: all lib tools oracle clean
