# Builds the state lattice planner checker and, when the reference tree is present, the reference's own
# src/state_lattice_planner.cpp against the header shims.  Outputs are git-ignored.  Usage: make -C oracle -f slp.mk
#   lib/liboracle_slp.so  crb_oracle_slp.c (the samplers and the lookup-table search restated) with crb_oracle.c for
#                         the restated sinf / cosf; loaded by oracle/slp.py, which runs generate_path's optimizer
#                         through liboracle_mptg.so (oracle/mptg.mk)
#   _ref/libref_slp.so    shim/ref_wrap_slp.cpp, which #includes the reference file from where it lies with main()
#                         renamed (nothing of it is copied here), with mptg.mk's flags and include order: -w because
#                         calc_diff narrows double to float in a brace-init; shim_mptg/ first for its Eigen stand-in
CC      := gcc
CXX     := g++
# the flags of liboracle.so (see Makefile): no implicit contraction; -mfma only turns fma() calls into the instruction
FMAFLAG := $(shell grep -q -m1 ' fma ' /proc/cpuinfo && echo -mfma)
CFLAGS  ?= -O2 -ffp-contract=off -fPIC -fopenmp -Wall -Wextra -std=c11 $(FMAFLAG)
REF     ?= /root/reference
REF_SLP := $(REF)/src/state_lattice_planner.cpp

all: lib/liboracle_slp.so ref_slp

lib/liboracle_slp.so: crb_oracle_slp.c crb_oracle.c crb_oracle_slp.h crb_oracle.h ../include/crb.h
	@mkdir -p lib
	$(CC) $(CFLAGS) -shared -o $@ crb_oracle_slp.c crb_oracle.c -lm

ref_slp:
	@if [ -f "$(REF_SLP)" ]; then mkdir -p _ref && \
	  $(CXX) -std=c++11 -O2 -ffp-contract=off -fPIC -shared -w -Ishim_mptg -Ishim -I$(REF)/include \
	    -DREF_SRC="\"$(REF_SLP)\"" shim/ref_wrap_slp.cpp -o _ref/libref_slp.so && echo "oracle/_ref: libref_slp.so built"; \
	 else echo "reference tree absent: skipping oracle/_ref/libref_slp.so"; fi

.PHONY: all ref_slp
