# Builds the dynamic-window-approach checker and, when the reference tree is present, the reference's own
# src/dynamic_window_approach.cpp against the header shims.  Outputs are git-ignored.  Usage: make -C oracle -f dwa.mk
#   lib/liboracle_dwa.so  crb_oracle_dwa.c (dwa_control, motion, acosf restated) with crb_oracle.c for the
#                         restated sinf / cosf; loaded by oracle/dwa.py
#   _ref/libref_dwa.so    shim/ref_wrap_dwa.cpp, which #includes the reference file from where it lies (nothing of it
#                         is copied here) after <algorithm> and <limits>: the file uses std::max and
#                         std::numeric_limits and relies on real OpenCV's headers to bring them in
CC      := gcc
CXX     := g++
# the flags of liboracle.so (see Makefile): no implicit contraction; -mfma only turns fma() calls into the instruction
FMAFLAG := $(shell grep -q -m1 ' fma ' /proc/cpuinfo && echo -mfma)
CFLAGS  ?= -O2 -ffp-contract=off -fPIC -fopenmp -Wall -Wextra -std=c11 $(FMAFLAG)
REF     ?= /root/reference
REF_DWA := $(REF)/src/dynamic_window_approach.cpp

all: lib/liboracle_dwa.so ref_dwa

lib/liboracle_dwa.so: crb_oracle_dwa.c crb_oracle.c crb_oracle_dwa.h crb_oracle.h ../include/crb.h
	@mkdir -p lib
	$(CC) $(CFLAGS) -shared -o $@ crb_oracle_dwa.c crb_oracle.c -lm

# the same compiler flags as shim/build_ref.sh uses for the other reference programs
ref_dwa:
	@if [ -f "$(REF_DWA)" ]; then mkdir -p _ref && \
	  $(CXX) -std=c++11 -O2 -ffp-contract=off -fPIC -shared -w -Ishim -I$(REF)/include \
	    -DREF_SRC="\"$(REF_DWA)\"" shim/ref_wrap_dwa.cpp -o _ref/libref_dwa.so && echo "oracle/_ref: libref_dwa.so built"; \
	 else echo "reference tree absent: skipping oracle/_ref/libref_dwa.so"; fi

.PHONY: all ref_dwa
