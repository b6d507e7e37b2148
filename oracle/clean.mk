# Builds the CPU checker of the surface clean and triangle filter (test infrastructure; never linked into the
# product). Integer and copy work only, but the same flags as the other checkers.
CC ?= gcc
CFLAGS = -O2 -fPIC -shared -std=c11 -Wall -ffp-contract=off

all: libclean.so

libclean.so: clean.c
	$(CC) $(CFLAGS) -o $@ clean.c -lm

clean:
	rm -f libclean.so
