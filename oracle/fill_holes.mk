# Builds the CPU checker of the surface hole filler (test infrastructure; never linked into the product).
# -ffp-contract=off: no fused multiply-add, so the double arithmetic is the one the contract states.
CC ?= gcc
CFLAGS = -O2 -fPIC -shared -std=c11 -Wall -ffp-contract=off

all: libfill_holes.so

libfill_holes.so: fill_holes.c
	$(CC) $(CFLAGS) -o $@ fill_holes.c -lm

clean:
	rm -f libfill_holes.so
