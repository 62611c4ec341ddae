# Builds the automatic sync-point module of the CPU oracle (TEST INFRASTRUCTURE; never linked into the product).  Stand-alone: it needs
# nothing from libgf_oracle.so.  Same flags as oracle/Makefile: strict IEEE, no FMA contraction, no fast-math.
CC      ?= gcc
CFLAGS  := -O2 -std=c11 -fPIC -ffp-contract=off -fno-fast-math -fexcess-precision=standard -Wall -Wextra -Wno-unused-parameter

all: libgf_oracle_optsync.so

libgf_oracle_optsync.so: gf_oracle_optsync.c
	$(CC) $(CFLAGS) -shared -o $@ gf_oracle_optsync.c -lm

clean:
	rm -f libgf_oracle_optsync.so
.PHONY: all clean
