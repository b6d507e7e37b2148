# Builds the CPU checker of "Remove non-visible faces" (test infrastructure; never linked into the product).
# Same flags as the other checkers: -ffp-contract=off, so every float64 step rounds as the device's does.
CC ?= gcc
CFLAGS = -O2 -fPIC -shared -std=c11 -ffp-contract=off -fno-fast-math -Wall -Wno-unused-function

all: libvisibility.so

libvisibility.so: visibility.c
	$(CC) $(CFLAGS) -o $@ visibility.c -lm

clean:
	rm -f libvisibility.so
