# Builds the LQR path-tracking checker and, when the reference tree is present, the LQR programs' own functions
# against the header shims.  Outputs are git-ignored.  Usage: make -C oracle -f lqrt.mk
#   lib/liboracle_lqrt.so   crb_oracle_lqrt.c (calc_nearest_index, lqr_steering_control and update of both LQR
#                           programs restated) with crb_oracle.c for solve_DARE + dlqr; loaded by oracle/lqrt.py
#   _ref/libref_lqrt4.so    shim/ref_wrap_lqrt.cpp around src/lqr_steer_control.cpp, and _ref/libref_lqrt5.so around
#                           src/lqr_speed_steer_control.cpp: the reference files are #included from where they lie
#                           (nothing of them is copied here), with the flags of shim/build_ref.sh
CC      := gcc
CXX     := g++
# the flags of liboracle.so (see Makefile): no implicit contraction; -mfma only turns fma() calls into the instruction
FMAFLAG := $(shell grep -q -m1 ' fma ' /proc/cpuinfo && echo -mfma)
CFLAGS  ?= -O2 -ffp-contract=off -fPIC -fopenmp -Wall -Wextra -std=c11 $(FMAFLAG)
REF     ?= /root/reference
REFFLAGS := -std=c++11 -O2 -ffp-contract=off -fPIC -shared -w -Ishim -I$(REF)/include

all: lib/liboracle_lqrt.so ref_lqrt

lib/liboracle_lqrt.so: crb_oracle_lqrt.c crb_oracle.c crb_oracle_lqrt.h crb_oracle.h
	@mkdir -p lib
	$(CC) $(CFLAGS) -shared -o $@ crb_oracle_lqrt.c crb_oracle.c -lm

ref_lqrt: shim/ref_wrap_lqrt.cpp
	@if [ -f "$(REF)/src/lqr_steer_control.cpp" ] && [ -f "$(REF)/src/lqr_speed_steer_control.cpp" ]; then \
	  mkdir -p _ref && \
	  $(CXX) $(REFFLAGS) -DWHICH=4 -DREF_SRC="\"$(REF)/src/lqr_steer_control.cpp\"" shim/ref_wrap_lqrt.cpp \
	    -o _ref/libref_lqrt4.so && \
	  $(CXX) $(REFFLAGS) -DWHICH=5 -DREF_SRC="\"$(REF)/src/lqr_speed_steer_control.cpp\"" shim/ref_wrap_lqrt.cpp \
	    -o _ref/libref_lqrt5.so && echo "oracle/_ref: libref_lqrt4.so libref_lqrt5.so built"; \
	 else echo "reference tree absent: skipping oracle/_ref/libref_lqrt*.so"; fi

.PHONY: all ref_lqrt
