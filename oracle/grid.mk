# Builds the grid A* / Dijkstra checker and, when the reference tree is present, the reference's own src/a_star.cpp
# and src/dijkstra.cpp against the header shims.  Outputs are git-ignored.  Usage: make -C oracle -f grid.mk
#   lib/liboracle_grid.so    crb_oracle_grid.c (the obstacle map and both searches restated); loaded by oracle/grid.py
#   _ref/libref_astar.so     shim_grid/ref_wrap_grid.cpp, which #includes the reference file from where it lies with main()
#   _ref/libref_dijkstra.so  renamed (nothing of it is copied here).  Two libraries: both files define Node and
#                            calc_final_path.  -w because the reference compares int with size_t.  shim_grid/ comes
#                            first: its opencv2/opencv.hpp adds cv::Point and a recording cv::rectangle to shim/'s.
CC      := gcc
CXX     := g++
# the flags of liboracle.so (see Makefile): no implicit contraction
FMAFLAG := $(shell grep -q -m1 ' fma ' /proc/cpuinfo && echo -mfma)
CFLAGS  ?= -O2 -ffp-contract=off -fPIC -fopenmp -Wall -Wextra -std=c11 $(FMAFLAG)
REF     ?= /root/reference
REF_ASTAR := $(REF)/src/a_star.cpp
REF_DIJKSTRA := $(REF)/src/dijkstra.cpp

all: lib/liboracle_grid.so ref_grid

lib/liboracle_grid.so: crb_oracle_grid.c crb_oracle_grid.h
	@mkdir -p lib
	$(CC) $(CFLAGS) -shared -o $@ crb_oracle_grid.c -lm

ref_grid: shim_grid/opencv2/opencv.hpp shim_grid/ref_wrap_grid.cpp
	@if [ -f "$(REF_ASTAR)" ] && [ -f "$(REF_DIJKSTRA)" ]; then mkdir -p _ref && \
	  $(CXX) -std=c++11 -O2 -ffp-contract=off -fPIC -shared -w -Ishim_grid -Ishim -I$(REF)/include \
	    -DREF_SRC="\"$(REF_ASTAR)\"" -DREF_PLAN=a_star_planning shim_grid/ref_wrap_grid.cpp -o _ref/libref_astar.so && \
	  $(CXX) -std=c++11 -O2 -ffp-contract=off -fPIC -shared -w -Ishim_grid -Ishim -I$(REF)/include \
	    -DREF_SRC="\"$(REF_DIJKSTRA)\"" -DREF_PLAN=dijkstra_star_planning shim_grid/ref_wrap_grid.cpp \
	    -o _ref/libref_dijkstra.so && echo "oracle/_ref: libref_astar.so libref_dijkstra.so built"; \
	 else echo "reference tree absent: skipping oracle/_ref/libref_astar.so and libref_dijkstra.so"; fi

.PHONY: all ref_grid
