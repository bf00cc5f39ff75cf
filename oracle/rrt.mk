# Builds the RRT checker and, when the reference tree is present, the reference's own include/rrt.h against the header
# shims.  Outputs are git-ignored.  Usage: make -C oracle -f rrt.mk
#   lib/liboracle_rrt.so  crb_oracle_rrt.c (mt19937, the two distributions, atan2f and RRT::planning restated) with
#                         crb_oracle.c for the restated sinf / cosf; loaded by oracle/rrt.py
#   _ref/libref_rrt.so    shim_rrt/ref_wrap_rrt.cpp, which #includes the reference header from where it lies (nothing
#                         of it is copied here).  -w because the header compares int with size_t.  shim_rrt/ comes
#                         first: its opencv2/opencv.hpp adds cv::Point and a cv::line that bounds the planner's loop.
CC      := gcc
CXX     := g++
# the flags of liboracle.so (see Makefile): no implicit contraction; -mfma only turns fma() calls into the instruction
FMAFLAG := $(shell grep -q -m1 ' fma ' /proc/cpuinfo && echo -mfma)
CFLAGS  ?= -O2 -ffp-contract=off -fPIC -fopenmp -Wall -Wextra -std=c11 $(FMAFLAG)
REF     ?= /root/reference
REF_RRT := $(REF)/include/rrt.h

all: lib/liboracle_rrt.so ref_rrt

lib/liboracle_rrt.so: crb_oracle_rrt.c crb_oracle.c crb_oracle_rrt.h crb_oracle.h
	@mkdir -p lib
	$(CC) $(CFLAGS) -shared -o $@ crb_oracle_rrt.c crb_oracle.c -lm

ref_rrt: shim_rrt/opencv2/opencv.hpp shim_rrt/ref_wrap_rrt.cpp
	@if [ -f "$(REF_RRT)" ]; then mkdir -p _ref && \
	  $(CXX) -std=c++11 -O2 -ffp-contract=off -fPIC -shared -w -Ishim_rrt -Ishim -I$(REF)/include \
	    shim_rrt/ref_wrap_rrt.cpp -o _ref/libref_rrt.so && echo "oracle/_ref: libref_rrt.so built"; \
	 else echo "reference tree absent: skipping oracle/_ref/libref_rrt.so"; fi

.PHONY: all ref_rrt
