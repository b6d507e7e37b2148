# Builds the CPU checker of surface normals and mass properties (test infrastructure; never linked into the
# product). -ffp-contract=off: no fused multiply-add, so the arithmetic is the one the contract states.
CC ?= gcc
CFLAGS = -O2 -fPIC -shared -std=c11 -Wall -ffp-contract=off -fno-fast-math

all: libnormals.so

libnormals.so: normals.c
	$(CC) $(CFLAGS) -o $@ normals.c -lm

clean:
	rm -f libnormals.so
