# Builds the CPU checker of the volume rendering's data preparation (test infrastructure; never linked into the
# product). -ffp-contract=off: no fused multiply-add, so the arithmetic is the one the contract states.
CC ?= gcc
CFLAGS = -O2 -fPIC -shared -std=c11 -Wall -ffp-contract=off -fno-fast-math

all: libraycasting.so

libraycasting.so: raycasting.c
	$(CC) $(CFLAGS) -o $@ raycasting.c -lm

clean:
	rm -f libraycasting.so
