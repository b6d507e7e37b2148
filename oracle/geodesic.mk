# Builds the CPU checker of the geodesic surface measurement (test infrastructure; never linked into the
# product). -ffp-contract=off: no fused multiply-add, so the arithmetic is the one the contract states.
CC ?= gcc
CFLAGS = -O2 -fPIC -shared -std=c11 -Wall -ffp-contract=off -fno-fast-math

all: libgeodesic.so

libgeodesic.so: geodesic.c
	$(CC) $(CFLAGS) -o $@ geodesic.c -lm

clean:
	rm -f libgeodesic.so
