# Builds the visual-features sync module of the CPU oracle (TEST INFRASTRUCTURE; never linked into the product) on top of libgf_oracle.so.
# Same flags as oracle/Makefile: strict IEEE, no FMA contraction, no fast-math.
CC      ?= gcc
CFLAGS  := -O2 -std=c11 -fPIC -ffp-contract=off -fno-fast-math -fexcess-precision=standard -Wall -Wextra -Wno-unused-parameter -Wno-misleading-indentation

all: libgf_oracle_sync.so

libgf_oracle.so:
	$(MAKE) -f Makefile libgf_oracle.so

libgf_oracle_sync.so: gf_oracle_sync.c gf_oracle_sync.h gf_oracle.h ../include/gyroflow_cuda.h libgf_oracle.so
	$(CC) $(CFLAGS) -shared -o $@ gf_oracle_sync.c -L. -l:libgf_oracle.so -Wl,-rpath,'$$ORIGIN' -lm -lpthread

clean:
	rm -f libgf_oracle_sync.so
.PHONY: all clean
