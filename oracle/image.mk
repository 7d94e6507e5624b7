# Builds the image post-processing oracle (orc_image.c) on its own; same flags as oracle/Makefile (the reference's
# Release defaults, -ffp-contract=off pins "no FMA").  Test infrastructure only.
CC := /usr/bin/gcc
CFLAGS = -O3 -DNDEBUG -std=c11 -fPIC -ffp-contract=off -Wall -Wextra -Wno-unused-parameter

all: libouster_oracle_image.so

libouster_oracle_image.so: orc_image.c orc_image_t.h
	$(CC) $(CFLAGS) -shared -o $@ orc_image.c -lm

clean:
	rm -f libouster_oracle_image.so
