# Builds the CPU checker of the surface connectivity tools (test infrastructure; never linked into the product).
CC ?= gcc
CFLAGS = -O2 -fPIC -shared -std=c11 -Wall

all: libconnectivity.so

libconnectivity.so: connectivity.c
	$(CC) $(CFLAGS) -o $@ connectivity.c

clean:
	rm -f libconnectivity.so
