# Builds the jump-flooding CPU checker (test infrastructure; never linked into the product).
# Same flags as the other checkers: -ffp-contract=off, the reference (Rust) never fuses multiply-add.
CC ?= gcc
CFLAGS = -O2 -fPIC -shared -std=c11 -ffp-contract=off -fno-fast-math -Wall -Wno-unused-function

all: libvoronoi.so

libvoronoi.so: voronoi.c
	$(CC) $(CFLAGS) -o $@ voronoi.c -lm -lpthread

clean:
	rm -f libvoronoi.so
