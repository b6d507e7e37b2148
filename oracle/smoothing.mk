# Builds the CPU checker of the Laplacian surface smoothing (test infrastructure; never linked into the product).
# -ffp-contract=off: no fused multiply-add, so the double arithmetic is the one the contract states.
CC ?= gcc
CFLAGS = -O2 -fPIC -shared -std=c11 -Wall -ffp-contract=off

all: libsmoothing.so

libsmoothing.so: smoothing.c
	$(CC) $(CFLAGS) -o $@ smoothing.c -lm

clean:
	rm -f libsmoothing.so
