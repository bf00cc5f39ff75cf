# Builds the model-predictive trajectory generation checker and, when the reference tree is present, the
# reference's own include/trajectory_optimizer.h against the header shims.  Outputs are git-ignored.
# Usage: make -C oracle -f mptg.mk
#   lib/liboracle_mptg.so  crb_oracle_mptg.c (optimizer_traj, MotionModel and tanf restated) with crb_oracle.c for
#                          the restated sinf / cosf; loaded by oracle/mptg.py
#   _ref/libref_mptg.so    shim/ref_wrap_mptg.cpp, which #includes the reference header from where it lies (nothing
#                          of it is copied here); -w because calc_diff narrows double to float in a brace-init.
#                          shim_mptg/ comes first: its Eigen stand-in has the operator[], column-vector comma
#                          initialisation and 3x3 inverse these headers use; OpenCV's stand-in comes from shim/
CC      := gcc
CXX     := g++
# the flags of liboracle.so (see Makefile): no implicit contraction; -mfma only turns fma() calls into the instruction
FMAFLAG := $(shell grep -q -m1 ' fma ' /proc/cpuinfo && echo -mfma)
CFLAGS  ?= -O2 -ffp-contract=off -fPIC -fopenmp -Wall -Wextra -std=c11 $(FMAFLAG)
REF     ?= /root/reference
REF_MPTG := $(REF)/include/trajectory_optimizer.h

all: lib/liboracle_mptg.so ref_mptg

lib/liboracle_mptg.so: crb_oracle_mptg.c crb_oracle.c crb_oracle_mptg.h crb_oracle.h ../include/crb.h
	@mkdir -p lib
	$(CC) $(CFLAGS) -shared -o $@ crb_oracle_mptg.c crb_oracle.c -lm

# the same compiler flags as shim/build_ref.sh uses for the other reference programs
ref_mptg:
	@if [ -f "$(REF_MPTG)" ]; then mkdir -p _ref && \
	  $(CXX) -std=c++11 -O2 -ffp-contract=off -fPIC -shared -w -Ishim_mptg -Ishim -I$(REF)/include \
	    -DREF_HDR="\"$(REF_MPTG)\"" shim/ref_wrap_mptg.cpp -o _ref/libref_mptg.so && echo "oracle/_ref: libref_mptg.so built"; \
	 else echo "reference tree absent: skipping oracle/_ref/libref_mptg.so"; fi

.PHONY: all ref_mptg
